"""U on the GPU, path by path: the resident complete trie (kind 0) and the sparse resident secure trie (kind 1) against the
oracle after every update, at the RLP length edges of their nodes, across both update paths of kind 0 and both arena layouts
of kind 1, with the leaf-reference cache in play, and over the exact update sequences bench.py times (C4, C4 sparse).

Kind 0 has two leaf stages in front of one branch-level path: the fused one (host pointers, every value <= 512 bytes:
encode in shared memory, hash, store; it hashes nothing through the batched Keccak kernels, so keccak_msgs stays 0) and the
general one (device pointers, or a larger value: the leaves through the batched kernels, n_dirty messages).  The branch
levels are hashed in shared memory on both, so they add no messages.  Each kind-0 test checks the stats so that it cannot
drift onto the other path unnoticed."""
import numpy as np
import pytest

import oracle_lib

pytestmark = pytest.mark.gpu

E_INVALID = -1
FUSED_MAX_VALUE = 512  # the fused path's staging slot holds a leaf with a value up to this size


@pytest.fixture(scope="module")
def ctx():
    from phant_b200 import gpu
    c = gpu.Context(0)
    yield c
    c.close()


def _mem_available_gb():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) / 2 ** 20
    return 0.0


# ------------------------------------------------------------------------------------------------------------- kind 0
def keys_at(rng, pos, depth):
    """random 32-byte keys whose first `depth` nibbles spell the leaf positions `pos`"""
    pos = np.asarray(pos, np.uint64)
    keys = rng.integers(0, 256, (len(pos), 32), dtype=np.uint8)
    top = np.zeros((len(pos), 4), np.uint8)              # the first 8 nibbles, position left-aligned
    shifted = pos << np.uint64(32 - 4 * depth)
    for b in range(4):
        top[:, b] = ((shifted >> np.uint64(24 - 8 * b)) & np.uint64(0xff)).astype(np.uint8)
    nb = (depth + 1) // 2                                 # bytes that hold position nibbles
    keys[:, :nb] = top[:, :nb]
    if depth % 2:                                         # the last position byte keeps a random low nibble
        keys[:, nb - 1] |= rng.integers(0, 16, len(pos), dtype=np.uint8)
    return np.ascontiguousarray(keys)


def leaf_len(vl, depth, first=0xff):
    """bytes of rlp([hp(64 - depth nibbles, leaf), value]) for a value of vl bytes (first byte `first`)"""
    def hdr(n):
        return 1 if n <= 55 else 1 + (n.bit_length() + 7) // 8
    hpn = 1 + (64 - depth) // 2
    s_hp = 1 if hpn == 1 else 1 + hpn
    s_v = 1 if vl == 1 and first < 0x80 else hdr(vl) + vl
    payload = s_hp + s_v
    return hdr(payload) + payload


def edge_lengths(depth):
    """value lengths at the fused leaf kernel's edges for this depth"""
    out = {0, 1, 55, 56, 255, 256} | set(range(505, FUSED_MAX_VALUE + 1))
    for vl in range(0, FUSED_MAX_VALUE + 1):
        n = leaf_len(vl, depth)
        payload = n - (1 if n - 1 <= 55 else 1 + ((n - 1).bit_length() + 7) // 8)
        if n % 136 in (0, 1, 135) or payload in (55, 56, 255, 256, 257):
            out.add(vl)
        if vl and leaf_len(vl - 1, depth) != n - 1:          # the list header grows by a byte here
            out.update((vl - 1, vl))
    return sorted(out)


def vals_csr(vals):
    return oracle_lib.csr(vals, np.uint32)


def upd(ctx, t, o, keys, vals, path):
    """one update on the GPU trie `t` and on the oracle `o`; path = "fused" | "general" | "device" (general, device pointers);
    asserts the root and the stats witness of the path, returns the root"""
    from phant_b200 import gpu
    import torch
    depth = t_depth(t)
    flat = np.ascontiguousarray(keys.reshape(-1))
    v, voff = vals_csr(vals)
    ctx.reset_stats()
    if path == "device":
        ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
        try:
            dk, dv, do = (torch.from_numpy(np.array(a)).cuda() for a in (flat, v, voff.view(np.int32)))
            torch.cuda.synchronize()
            root = t.update(dk, dv, do, len(vals))
        finally:
            ctx.set_flags(0)
    else:
        root = t.update(flat, v, voff, len(vals))
    msgs = ctx.stats()["keccak_msgs"]
    if path == "fused":
        assert max(len(x) for x in vals) <= FUSED_MAX_VALUE
        assert msgs == 0, "fused path expected"
    else:
        assert path == "device" or max(len(x) for x in vals) > FUSED_MAX_VALUE
        assert msgs == len(vals), "general path expected"
    want = o.update(flat, vals)
    assert root == want, (path, depth, len(vals))
    assert t.root() == root
    return root


_depths = {}


def t_depth(t):
    return _depths[id(t)]


def open_pair(ctx, oracle, depth):
    t = ctx.trie_open(depth)
    _depths[id(t)] = depth
    o = oracle.ctrie(depth)
    assert t.root() == o.root(), depth
    return t, o


def rvals(rng, lengths):
    return [rng.integers(0, 256, int(n), dtype=np.uint8).tobytes() for n in lengths]


@pytest.mark.parametrize("depth", [1, 2, 3, 4, 5, 6])
def test_fused_leaf_value_length_sweep(ctx, oracle, depth):
    """every value length at an RLP or Keccak-block edge of the fused leaf kernel: empty value, one byte below and at 0x80,
    the 55/56 string and list header edges, leaves on a multiple of 136 bytes and one byte either side, the 1- to 2-byte
    length edge at 256 (0xb9 value / 0xf9 list header), and 505..512 (at depth 1 a 544..551-byte leaf: the last Keccak block
    holds padding only or a masked tail)"""
    rng = np.random.default_rng(100 + depth)
    lengths = edge_lengths(depth)
    vals = rvals(rng, lengths)
    vals[lengths.index(1)] = b"\x05"
    vals += [b"\x80", b"\x7f", b"\x00"]
    assert depth != 1 or {leaf_len(505, 1), leaf_len(512, 1)} == {544, 551}
    t, o = open_pair(ctx, oracle, depth)
    per = 16 if depth == 1 else len(vals)               # distinct positions: depth 1 has only 16
    for i in range(0, len(vals), per):
        chunk = vals[i:i + per]
        pos = rng.choice(16 ** depth, size=len(chunk), replace=False)
        upd(ctx, t, o, keys_at(rng, pos, depth), chunk, "fused")
    t.close()


def test_general_leaf_stage_host_and_device_pointers(ctx, oracle):
    """values up to ~5,000 bytes mixed with small ones: a value over 512 bytes sends a host-pointer update's leaves through the
    general stage; device pointers always take it.  Two tries of one seed get the same sequence, one from host memory and one from
    device memory, some updates fused on the host side; every root equals the oracle's"""
    for depth in (1, 3, 5):
        rng = np.random.default_rng(200 + depth)
        th, oh = open_pair(ctx, oracle, depth)
        td, od = open_pair(ctx, oracle, depth)
        for step in range(4):
            n = 16 if depth == 1 else 700
            pos = rng.choice(16 ** depth, size=n, replace=False)
            keys = keys_at(rng, pos, depth)
            lens = rng.choice([0, 1, 33, 56, 256, 511, 512, 513, 1000, 2020, 4999, 5000], size=n)
            if step % 2:
                lens = np.minimum(lens, FUSED_MAX_VALUE)
            else:
                lens[0] = 5000
            vals = rvals(rng, lens)
            r1 = upd(ctx, th, oh, keys, vals, "fused" if step % 2 else "general")
            r2 = upd(ctx, td, od, keys, vals, "device")
            assert r1 == r2
        th.close()
        td.close()


@pytest.mark.parametrize("depth", [4, 6])
def test_update_sequences_alternate_leaf_stages(ctx, oracle, depth):
    """12 successive updates on one trie; each reuses positions of earlier ones, and the largest value crosses 512 bytes
    every other update, so consecutive updates alternate between the fused and the general leaf stage"""
    rng = np.random.default_rng(300 + depth)
    t, o = open_pair(ctx, oracle, depth)
    seen = np.zeros(0, np.int64)
    for step in range(12):
        n = int(rng.integers(1, 4000))
        old = rng.choice(seen, size=min(len(seen), n // 2), replace=False) if len(seen) else seen
        pos = rng.permutation(np.unique(np.concatenate([old, rng.choice(16 ** depth, size=n, replace=False)])))
        seen = np.unique(np.concatenate([seen, pos]))
        general = step % 2 == 1
        lens = rng.integers(0, 700 if general else FUSED_MAX_VALUE + 1, len(pos))
        if general:
            lens[int(rng.integers(0, len(pos)))] = 600
        upd(ctx, t, o, keys_at(rng, pos, depth), rvals(rng, lens), "general" if general else "fused")
    t.close()


def test_refused_updates_leave_the_trie_unchanged_on_every_leaf_stage(ctx, oracle):
    """two dirty keys on one leaf position -- a repeated key, or two keys sharing their first `depth` nibbles -- make the
    update E_INVALID whichever leaf stage it takes; the root is unchanged, and the next update matches an oracle that never
    saw the refused one.  n_dirty = 0 returns the current root."""
    from phant_b200 import gpu
    import torch
    depth = 3
    rng = np.random.default_rng(400)
    t, o = open_pair(ctx, oracle, depth)
    upd(ctx, t, o, keys_at(rng, rng.choice(16 ** depth, 500, replace=False), depth), rvals(rng, rng.integers(0, 100, 500)), "fused")
    for path in ("fused", "general", "device"):
        for dup in ("repeat", "prefix"):
            before = t.root()
            pos = rng.choice(16 ** depth, size=300, replace=False)
            keys = keys_at(rng, pos, depth)
            if dup == "repeat":
                keys[200] = keys[17]
            else:
                keys[200] = keys_at(rng, [pos[17]], depth)[0]
                assert (keys[200] != keys[17]).any()
            lens = rng.integers(0, 100, 300)
            if path != "fused":
                lens[5] = 2000
            vals = rvals(rng, lens)
            v, voff = vals_csr(vals)
            flat = np.ascontiguousarray(keys.reshape(-1))
            with pytest.raises(gpu.PhantGpuError) as e:
                if path == "device":
                    ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
                    try:
                        dk, dv, do = (torch.from_numpy(np.array(a)).cuda() for a in (flat, v, voff.view(np.int32)))
                        torch.cuda.synchronize()
                        t.update(dk, dv, do, 300)
                    finally:
                        ctx.set_flags(0)
                else:
                    t.update(flat, v, voff, 300)
            assert e.value.code == E_INVALID, (path, dup)
            assert t.root() == before == o.root(), (path, dup)
            # the next valid update (same positions, the colliding key dropped) is right
            keep = np.ones(300, bool)
            keep[200] = False
            nxt = [x for x, k in zip(vals, keep) if k]
            upd(ctx, t, o, keys[keep], nxt, path if path != "general" or max(len(x) for x in nxt) > FUSED_MAX_VALUE else "fused")
    assert t.update(np.zeros(32, np.uint8), np.zeros(1, np.uint8), np.zeros(1, np.uint32), 0) == o.root()
    t.close()


def test_depth7_full_size_open_and_updates(ctx, oracle):
    """depth 7 (16^7 leaves): the largest trie, whose open hashes a level of 16^6 branches in one frontier launch; one
    100k fused update and one general update against the oracle's full-size trie"""
    need = 24
    if _mem_available_gb() < need:
        pytest.skip(f"the depth-7 oracle holds 8.6 GB of hashes; {need} GB of available host memory required")
    depth = 7
    rng = np.random.default_rng(700)
    t, o = open_pair(ctx, oracle, depth)
    pos = rng.choice(16 ** depth, size=100_000, replace=False)
    upd(ctx, t, o, keys_at(rng, pos, depth), rvals(rng, np.full(100_000, 78)), "fused")
    pos = rng.choice(16 ** depth, size=20_000, replace=False)
    lens = rng.integers(0, 200, 20_000)
    lens[0] = 1500
    upd(ctx, t, o, keys_at(rng, pos, depth), rvals(rng, lens), "general")
    t.close()
    del o


class _RecordingTrie:
    """forwards to a resident trie and keeps a host copy of every update's inputs with the root it returned"""

    def __init__(self, trie, log):
        self.trie, self.log = trie, log

    def update(self, keys32, leaf_vals, val_off, n_dirty):
        root = self.trie.update(keys32, leaf_vals, val_off, n_dirty)
        host = [np.array(a.cpu().numpy() if hasattr(a, "cpu") else a).reshape(-1) for a in (keys32, leaf_vals, val_off)]
        self.log.append((*host, int(n_dirty), root))
        return root

    def __getattr__(self, name):
        return getattr(self.trie, name)


class _RecordingContext:
    """a Context whose tries record their updates: bench.py's own C4 functions run on it unchanged, and the test then replays
    exactly what they applied"""

    def __init__(self, ctx):
        self.ctx, self.log = ctx, []

    def trie_open(self, *a, **kw):
        return _RecordingTrie(self.ctx.trie_open(*a, **kw), self.log)

    def __getattr__(self, name):
        return getattr(self.ctx, name)


def _run_bench_config(ctx, fn, steps, monkeypatch):
    import bench
    import torch
    from phant_b200 import gpu
    monkeypatch.delenv("PHANT_BENCH_SPARSE_KEYS", raising=False)   # the default size, as bench.py runs it
    rec = _RecordingContext(ctx)
    out = getattr(bench, fn)(rec, gpu, torch, torch.device("cuda", 0), steps)
    return rec.log, out


def test_c4_bench_sequence(ctx, oracle, monkeypatch):
    """bench.py's C4 run as bench.py runs it (bench_c4 on a recording context, six steps): the 16^6-leaf trie of the
    default seed, two warm-up sets, then the timed steps cycling the four 100k sets.  Every root it read back equals the
    oracle's full-size trie after the same update, and every update took the fused path bench.py means to time."""
    steps = 6
    log, out = _run_bench_config(ctx, "bench_c4", steps, monkeypatch)
    assert ctx.stats()["keccak_msgs"] == 0
    assert len(log) == 2 + steps and out["steps"] == steps
    depth = 6
    o = oracle.ctrie(depth)
    seen = set()
    for i, (keys, vals, voff, n, root) in enumerate(log):
        assert n == 100_000 and keys.size == 32 * n
        seen.add(keys[:32].tobytes())
        want = o.update(keys, [vals[int(voff[j]):int(voff[j + 1])].tobytes() for j in range(n)])
        assert root == want, i
    assert len(seen) == 4                                                # the four sets all ran


# ------------------------------------------------------------------------------------------------------------- kind 1
def _apply(trie, state, changes):
    """changes: {key32: value bytes (b"" deletes)} -> root after the update; `state` is the python-side model"""
    keys = list(changes)
    k = np.frombuffer(b"".join(keys), np.uint8)
    v, voff = oracle_lib.csr([changes[x] for x in keys], np.uint32)
    root = trie.update(k, v, voff, len(keys))
    for x in keys:
        if changes[x]:
            state[x] = changes[x]
        else:
            state.pop(x, None)
    return root


class Sparse:
    """a kind-1 trie with its Python model; every update is checked against oracle.mptize over the whole key set"""

    def __init__(self, ctx, oracle):
        self.ctx, self.oracle = ctx, oracle
        self.t = ctx.trie_open(0, kind=1)
        self.state = {}

    def apply(self, changes):
        self.ctx.reset_stats()
        root = _apply(self.t, self.state, changes)
        self.stats = self.ctx.stats()
        assert root == self.oracle.mptize(sorted(self.state.items())), len(self.state)
        assert self.t.root() == root
        return root


def key_in(rng, prefix_nibbles):
    """a random key starting with the given nibbles"""
    k = bytearray(rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
    for i, x in enumerate(prefix_nibbles):
        k[i >> 1] = (k[i >> 1] & 0x0f) | (x << 4) if i % 2 == 0 else (k[i >> 1] & 0xf0) | x
    return bytes(k)


def nibbles(key, n):
    return tuple((key[i >> 1] >> 4) if i % 2 == 0 else (key[i >> 1] & 15) for i in range(n))


def partial_top_keys(rng, L, per_bucket):
    """keys for a dense top of L levels whose level-(L-1) nodes have every child count from 2 to 16: node q keeps
    2 + q % 15 of its 16 buckets; returns {bucket nibbles: [keys]}"""
    buckets = {}
    for q in range(16 ** (L - 1)):
        up = tuple((q >> (4 * (L - 2 - i))) & 15 for i in range(L - 1))
        for c in rng.choice(16, size=2 + q % 15, replace=False):
            b = up + (int(c),)
            buckets[b] = [key_in(rng, b) for _ in range(per_bucket)]
    return buckets


def rval(rng, lo=1, hi=120):
    return rng.integers(0, 256, int(rng.integers(lo, hi)), dtype=np.uint8).tobytes()


@pytest.mark.parametrize("L,per_bucket", [(2, 40), (3, 32)])
def test_sparse_partial_dense_top(ctx, oracle, L, per_bucket):
    """dense-top nodes with 2..16 children (the 0xf8 list header for 2..7, absent children as 0x80); value updates through
    the partial path; whole buckets deleted; a node taken down to one child (the premise fails: the update must fall back to
    L - 1 dense levels and rebuild everything); emptied buckets filled again; at L = 3, a shrink by exactly one L step, so the
    partial path runs over thinned buckets"""
    rng = np.random.default_rng(500 + L)
    s = Sparse(ctx, oracle)
    buckets = partial_top_keys(rng, L, per_bucket)
    n = sum(len(v) for v in buckets.values())
    assert 16 ** (L + 2) > n >= 16 ** (L + 1), n             # 16..255 keys per bucket: L dense levels
    s.apply({k: rval(rng) for ks in buckets.values() for k in ks})
    # value updates in a few buckets: partial path, parents with partial masks re-hashed
    some = [b for i, b in enumerate(sorted(buckets)) if i % 7 == 0]
    s.apply({k: rval(rng) for b in some for k in buckets[b][:5]})
    # delete a whole bucket under every node that keeps >= 2 children afterwards
    parents = {}
    for b in buckets:
        parents.setdefault(b[:-1], []).append(b)
    gone = [sorted(v)[0] for v in parents.values() if len(v) >= 3][:6]
    s.apply({k: b"" for b in gone for k in buckets[b]})
    # fill them again
    s.apply({k: rval(rng) for b in gone for k in buckets[b]})
    if L == 3:
        # shrink by one L step: keep ~40% of every bucket (n drops below 16^4 keys), delete one more bucket in the same update
        drop = {}
        for b, ks in buckets.items():
            for k in ks[int(len(ks) * 0.4) + 1:]:
                drop[k] = b""
        extra = sorted(parents[sorted(parents)[5]])
        assert len(extra) >= 3
        drop.update({k: b"" for k in buckets[extra[0]]})
        s.apply(drop)
        assert 16 ** 4 > len(s.state) >= 16 ** 3
        s.apply({k: rval(rng) for k in list(s.state)[::50]})
    # a node with exactly two children loses one: single-child dense node -> fallback to L - 1
    two = [v for v in parents.values() if len(v) == 2][0]
    victim = [k for k in s.state if nibbles(k, L) == two[0]]
    assert victim
    n_before = len({nibbles(k, L) for k in s.state})
    s.apply({k: b"" for k in victim})
    assert s.stats["keccak_msgs"] >= n_before // 2, "the single-child fallback re-hashes every bucket"
    s.apply({k: rval(rng) for k in list(s.state)[::13]})
    s.t.close()


def test_sparse_value_sizes_and_layouts(ctx, oracle):
    """values at RLP edges and around the slot layout's 3,072-byte bound: a rebuild with every value <= 3,072 bytes takes the
    slot layout (hashed through fixed slots: no keccak_bytes), one with a larger value the CSR layout (keccak_bytes > 0); the
    same bucket switches layout between consecutive updates, so leaf-cache rows written under one layout are read under the
    other; deep key pairs that differ in the last nibble only give embedded leaves next to CSR-sized values"""
    rng = np.random.default_rng(600)
    s = Sparse(ctx, oracle)
    sizes = [1, 31, 32, 33, 55, 56, 255, 256, 3072, 3073, 9000]
    keys = [key_in(rng, ()) for _ in range(1500)]                     # L = 1: 16 buckets of ~94 keys
    base = {k: rval(rng, 1, 3073) for k in keys}
    for i, sz in enumerate(sizes):
        base[keys[i]] = rng.integers(0, 256, sz, dtype=np.uint8).tobytes()
    s.apply(base)
    assert s.stats["keccak_bytes"] > 0                                # 3073 and 9000: CSR
    bucket = nibbles(keys[0], 1)
    mine = [k for k in s.state if nibbles(k, 1) == bucket]
    # shrink every big value of this bucket and touch only it: slots
    s.apply({k: rval(rng, 1, 3073) for k in mine if len(s.state[k]) > 3072} | {mine[0]: b"\x01"})
    assert s.stats["keccak_bytes"] == 0, "slot layout expected"
    # the same bucket with a 9,000-byte value and an embedded-leaf pair: CSR
    pair = bytearray(key_in(rng, bucket))
    pair[31] = 0x10
    twin = bytearray(pair)
    twin[31] = 0x11
    s.apply({mine[1]: rng.integers(0, 256, 9000, dtype=np.uint8).tobytes(), bytes(pair): b"\x02", bytes(twin): b"\x03"})
    assert s.stats["keccak_bytes"] > 0, "CSR layout expected"
    # and back: slots, with every edge size but the big ones
    ch = {mine[1]: rng.integers(0, 256, 3072, dtype=np.uint8).tobytes()}
    for sz, k in zip(sizes[:9], mine[2:]):
        ch[k] = rng.integers(0, 256, sz, dtype=np.uint8).tobytes()
    s.apply(ch)
    assert s.stats["keccak_bytes"] == 0, "slot layout expected"
    # the CSR layout again in one bucket while another bucket builds in the same forest
    other = [k for k in s.state if nibbles(k, 1) != bucket][:3]
    s.apply({mine[3]: rng.integers(0, 256, 3073, dtype=np.uint8).tobytes(), other[0]: b"", other[1]: rval(rng)})
    assert s.stats["keccak_bytes"] > 0
    s.apply({bytes(pair): b"", mine[3]: b"\x7f"})
    s.t.close()


def test_sparse_leaf_cache(ctx, oracle):
    """the leaf-reference cache: a one-key value update in a bucket of b >= 16 keys hashes fewer than b messages (the other
    leaves come from the cache); an unchanged value whose leaf moves deeper or back up because a sibling was inserted or
    deleted is re-encoded, not served stale; a key deleted and re-inserted with the same value, then with another value"""
    rng = np.random.default_rng(601)
    s = Sparse(ctx, oracle)
    keys = [key_in(rng, ()) for _ in range(1000)]                     # L = 1, ~62 keys per bucket
    s.apply({k: rval(rng, 40, 120) for k in keys})
    k0 = keys[0]
    b = [k for k in s.state if nibbles(k, 1) == nibbles(k0, 1)]
    assert len(b) >= 16
    s.apply({k0: rval(rng, 40, 120)})
    assert 0 < s.stats["keccak_msgs"] < len(b), (s.stats["keccak_msgs"], len(b))
    # a sibling sharing 20 nibbles with k1: k1's leaf moves deeper, its value stays the same
    k1 = keys[1]
    sib = key_in(rng, nibbles(k1, 20) + (nibbles(k1, 21)[20] ^ 8,))
    s.apply({sib: rval(rng, 40, 120)})
    s.apply({sib: rval(rng, 40, 120)})                                # k1 deeper, served from its new cache row
    s.apply({sib: b""})                                               # and back up
    s.apply({k1: s.state[k1], keys[3]: rval(rng, 40, 120)})           # same value re-written: no change
    # delete, re-insert with the same value, then with another
    v = s.state[keys[4]]
    s.apply({keys[4]: b""})
    s.apply({keys[4]: v})
    s.apply({keys[4]: rval(rng, 40, 120)})
    s.t.close()


class _SortedModel:
    """the key set of a secure trie held in numpy: keys (n x 32, sorted) with fixed-size values (n x w).  Lookups go by the
    first 8 key bytes, which must be unique (they are, for random keys); every hit is confirmed on the whole key."""

    def __init__(self, width):
        self.w = width
        self.keys = np.zeros((0, 32), np.uint8)
        self.vals = np.zeros((0, width), np.uint8)
        self.pre = np.zeros(0, np.uint64)

    @staticmethod
    def _prefix(keys):
        return np.ascontiguousarray(keys[:, :8]).view(">u8").reshape(-1).astype(np.uint64)

    def apply(self, keys32, vals, val_off, n):
        """an update as the trie takes it: a w-byte value upserts, an empty one deletes"""
        keys = keys32.reshape(n, 32)
        off = val_off.astype(np.int64)
        lens = np.diff(off)
        assert set(np.unique(lens).tolist()) <= {0, self.w}
        put, gone = lens > 0, lens == 0
        rows = np.zeros((n, self.w), np.uint8)
        pi = np.nonzero(put)[0]
        if len(pi):
            starts = off[pi]
            if (starts == starts[0] + self.w * np.arange(len(pi))).all():   # one contiguous block: no index array
                rows[pi] = vals[starts[0]:starts[0] + self.w * len(pi)].reshape(-1, self.w)
            else:
                rows[pi] = vals[starts[:, None] + np.arange(self.w)[None, :]]
        pk = self._prefix(keys)
        idx = np.searchsorted(self.pre, pk)
        at = np.minimum(idx, max(len(self.pre) - 1, 0))
        found = (idx < len(self.pre)) & (self.pre[at] == pk) if len(self.pre) else np.zeros(n, bool)
        if found.any():
            assert (self.keys[at[found]] == keys[found]).all()
        self.vals[at[found & put]] = rows[found & put]
        new = ~found & put
        if (found & gone).any() or new.any():
            keep = np.ones(len(self.keys), bool)
            keep[at[found & gone]] = False
            keys_all = np.concatenate([self.keys[keep], keys[new]])
            vals_all = np.concatenate([self.vals[keep], rows[new]])
            pre = self._prefix(keys_all)
            order = np.argsort(pre, kind="stable")
            self.keys, self.vals, self.pre = keys_all[order], vals_all[order], pre[order]
            assert (np.diff(self.pre.astype(np.uint64)) > 0).all(), "8-byte key prefixes must be unique"

    def root(self, oracle):
        n = len(self.keys)
        koff = (np.arange(n + 1, dtype=np.uint64) * 32).astype(np.uint32)
        voff = np.arange(n + 1, dtype=np.uint64) * self.w
        return oracle.mptize_csr(self.keys.reshape(-1), koff, self.vals.reshape(-1), voff)


def test_c4_sparse_bench_sequence(ctx, oracle, monkeypatch):
    """bench.py's C4 sparse run as bench.py runs it (bench_c4_sparse on a recording context, three steps): the initial
    build of 16^6 random keys (L = 5), the warm-up upsert set, the three timed sets once each, then the 50k-insert /
    50k-delete step.  Every root it read back equals oracle.mptize over a numpy-held model of the key set."""
    need = 24
    if _mem_available_gb() < need:
        pytest.skip(f"the 16^6-key oracle trie (about 11 GB) and its model need {need} GB of available host memory")
    log, out = _run_bench_config(ctx, "bench_c4_sparse", 3, monkeypatch)
    assert len(log) == 1 + 1 + 3 + 1 and out["steps"] == 3
    assert log[0][3] == 16 ** 6
    model = _SortedModel(78)
    prev = None
    for i, (keys, vals, voff, n, root) in enumerate(log):
        before = model.vals.copy() if prev is not None else None
        model.apply(keys, vals, voff, n)
        same = before is not None and len(before) == len(model.vals) and (before == model.vals).all()
        if same:
            assert root == prev, i                                      # the warm-up set again: nothing changed
        else:
            assert root == model.root(oracle), i
        prev = root
    assert len(model.keys) == 16 ** 6                                   # 50k in, 50k out
