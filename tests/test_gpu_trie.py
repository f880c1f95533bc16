"""M / S / U on the GPU: trie roots bit-identical to the reference's vectors, the fixtures and the oracle."""
import numpy as np
import pytest

import oracle_lib
from helpers import index_trie_items

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    from phant_b200 import gpu
    c = gpu.Context(0)
    yield c
    c.close()


def gpu_mptize(ctx, kv):
    keys, koff = oracle_lib.csr([k for k, _ in kv], np.uint32)
    vals, voff = oracle_lib.csr([v for _, v in kv], np.uint64)
    return ctx.mpt_root(keys, koff, vals, voff, len(kv))


def test_mptize_reference_roots(ctx, golden):
    """src/mpt/mpt.zig:326-385 through the GPU builder (leaf root, embedded leaves, extension, branch value)."""
    for c in golden("mptize_kat.json")["cases"]:
        kv = [(bytes.fromhex(k), bytes.fromhex(v)) for k, v in c["kv"]]
        assert gpu_mptize(ctx, kv).hex() == c["root"], c["name"]


def test_evmone_topologies(ctx, golden):
    g = golden("evmone_mpt_kat.json")
    for grp in g["topologies"]:
        for upto in range(1, len(grp) + 1):
            kv = sorted((bytes.fromhex(e["key"]), bytes.fromhex(e["value"])) for e in grp[:upto])
            assert gpu_mptize(ctx, kv).hex() == grp[upto - 1]["root_after_insert"]
    for e in g["examples"]:
        kv = sorted((bytes.fromhex(k), bytes.fromhex(v)) for k, v in e["kv"])
        assert gpu_mptize(ctx, kv).hex() == e["root"], e["name"]


def test_fixture_list_roots(ctx, golden):
    """87 + 87 transaction / withdrawal index tries (src/blockchain/blockchain.zig:209-235), up to 400 items."""
    g = golden("fixture_states.json.gz")
    n = 0
    for t in g["tests"]:
        for b in t["blocks"]:
            txs = [bytes.fromhex(x) for x in b["tx_values"]]
            wds = [bytes.fromhex(x) for x in b["wd_values"]]
            assert gpu_mptize(ctx, index_trie_items(txs)).hex() == b["transactionsTrie"]
            assert gpu_mptize(ctx, index_trie_items(wds)).hex() == b["withdrawalsRoot"]
            n += 1
    assert n == 87


def random_prefixy_items(rng, n):
    """variable-length keys with many shared prefixes and keys that are prefixes of others; values 0..70 bytes"""
    keys = set()
    while len(keys) < n:
        base = bytes(rng.integers(0, 4, int(rng.integers(0, 5)), dtype=np.uint8))  # small alphabet -> collisions
        ext = bytes(rng.integers(0, 256, int(rng.integers(0, 4)), dtype=np.uint8))
        keys.add(base + ext)
    out = []
    for k in sorted(keys):
        vl = int(rng.choice([0, 1, 1, 2, 5, 20, 31, 32, 33, 55, 56, 70]))
        v = rng.integers(0, 256, vl, dtype=np.uint8).tobytes()
        if vl == 1 and rng.random() < 0.5:
            v = bytes([int(rng.integers(0, 0x80))])
        out.append((k, v))
    return out


def test_random_tries_vs_oracle(ctx, oracle):
    rng = np.random.default_rng(17)
    for n in [1, 2, 3, 5, 9, 17, 40, 100, 300, 1000]:
        for rep in range(3):
            kv = random_prefixy_items(rng, n)
            assert gpu_mptize(ctx, kv) == oracle.mptize(kv), (n, rep)


def test_big_values_and_long_keys(ctx, oracle):
    rng = np.random.default_rng(3)
    kv = sorted((bytes(rng.integers(0, 256, int(rng.integers(1, 80)), dtype=np.uint8)),
                 rng.integers(0, 256, int(rng.integers(0, 9000)), dtype=np.uint8).tobytes()) for _ in range(200))
    kv = [kv[i] for i in range(len(kv)) if i == 0 or kv[i][0] != kv[i - 1][0]]
    assert gpu_mptize(ctx, kv) == oracle.mptize(kv)


def test_unsorted_and_duplicates_rejected(ctx):
    from phant_b200 import gpu
    for kv in ([(b"\x02", b"a"), (b"\x01", b"b")], [(b"\x01", b"a"), (b"\x01", b"b")], [(b"\x01\x02", b"a"), (b"\x01", b"b")]):
        with pytest.raises(gpu.PhantGpuError) as e:
            gpu_mptize(ctx, kv)
        assert e.value.code == -1
    assert gpu_mptize(ctx, []).hex() == "56e81f171bcc55a6ff8345e692c0f86e5b48e01b996cadc001622fb5e363b421"


def test_large_secure_trie(ctx, oracle):
    rng = np.random.default_rng(23)
    n = 200_000
    keys = np.unique(rng.integers(0, 256, (n, 32), dtype=np.uint8), axis=0)
    keys = sorted(k.tobytes() for k in keys)
    vals = [rng.integers(0, 256, int(l), dtype=np.uint8).tobytes() for l in rng.integers(33, 110, len(keys))]
    kv = list(zip(keys, vals))
    assert gpu_mptize(ctx, kv) == oracle.mptize(kv)


# ---------------------------------------------------------------- S
def gpu_state_root(ctx, accounts):
    n = len(accounts)
    one = np.zeros(1, np.uint8)
    addr = np.frombuffer(b"".join(bytes.fromhex(a["address"]) for a in accounts), np.uint8) if n else one
    nonce = np.array([a["nonce"] for a in accounts], np.uint64) if n else np.zeros(1, np.uint64)
    bal = np.frombuffer(b"".join(bytes.fromhex(a["balance"]) for a in accounts), np.uint8) if n else one
    code, coff = oracle_lib.csr([bytes.fromhex(a["code"]) for a in accounts])
    sk, sv, soff = [], [], [0]
    for a in accounts:
        for k, v in a["storage"].items():
            sk.append(bytes.fromhex(k))
            sv.append(bytes.fromhex(v))
        soff.append(len(sk))
    skeys = np.frombuffer(b"".join(sk), np.uint8) if sk else one
    svals = np.frombuffer(b"".join(sv), np.uint8) if sv else one
    return ctx.state_root(n, addr, nonce, bal, code, coff, skeys, svals, np.array(soff, np.uint64))


def test_evmone_state_roots(ctx, golden):
    for s in golden("evmone_mpt_kat.json")["states"]:
        assert gpu_state_root(ctx, s["accounts"]).hex() == s["root"], s["name"]


def test_fixture_state_roots(ctx, golden):
    """the 84 + 84 roots the exec-spec fixtures pin (pre vs genesis stateRoot, postState vs last block's)"""
    g = golden("fixture_states.json.gz")
    roots = {k: gpu_state_root(ctx, v).hex() for k, v in g["tables"].items()}
    for t in g["tests"]:
        assert roots[t["pre"]] == t["pre_root"], (t["file"], t["name"], "pre")
        assert roots[t["post"]] == t["post_root"], (t["file"], t["name"], "post")


def test_random_state_vs_oracle(ctx, oracle):
    rng = np.random.default_rng(9)
    accounts = []
    for i in range(3000):
        ns = int(rng.choice([0, 0, 0, 1, 2, 5, 40]))
        storage = {}
        for _ in range(ns):
            k = rng.integers(0, 256, 32, dtype=np.uint8).tobytes().hex()
            v = bytes(32) if rng.random() < 0.15 else (bytes(int(rng.integers(0, 32))) + rng.integers(1, 256, 32, dtype=np.uint8).tobytes())[:32]
            storage[k] = v.hex()
        accounts.append({"address": rng.integers(0, 256, 20, dtype=np.uint8).tobytes().hex(), "nonce": int(rng.choice([0, 1, 127, 128, 70000])),
                         "balance": "%064x" % int(rng.choice([0, 1, 127, 128, 10**18, 2**255])),
                         "code": rng.integers(0, 256, int(rng.choice([0, 0, 10, 500, 3000])), dtype=np.uint8).tobytes().hex(),
                         "storage": storage})
    assert gpu_state_root(ctx, accounts) == oracle.state_root(accounts)


# ---------------------------------------------------------------- U
def keys_at_positions(rng, pos, depth):
    """random 32-byte keys whose first `depth` nibbles spell the leaf position"""
    keys = rng.integers(0, 256, (len(pos), 32), dtype=np.uint8)
    for i, p in enumerate(pos):
        for j in range(depth):
            nb = (int(p) >> (4 * (depth - 1 - j))) & 15
            b = int(keys[i, j >> 1])
            keys[i, j >> 1] = (b & 0x0f) | (nb << 4) if j % 2 == 0 else (b & 0xf0) | nb
    return keys


def test_resident_trie_small(ctx, oracle):
    for depth in (1, 3, 4):
        o = oracle.ctrie(depth)
        t = ctx.trie_open(depth)
        assert t.root() == o.root(), depth
        rng = np.random.default_rng(depth)
        n = 300 if depth >= 3 else 7
        pos = rng.choice(16 ** depth, size=min(n, 16 ** depth), replace=False)  # distinct leaf positions
        keys = keys_at_positions(rng, pos, depth)
        vals = [rng.integers(0, 256, int(l), dtype=np.uint8).tobytes() for l in rng.integers(1, 120, len(pos))]
        v, voff = oracle_lib.csr(vals, np.uint32)
        flat = np.ascontiguousarray(keys.reshape(-1))
        r1 = t.update(flat, v, voff, len(pos))
        assert r1 == o.update(flat, vals), depth
        assert t.update(flat, v, voff, len(pos)) == r1  # idempotent
        t.close()


def test_resident_trie_full_size(ctx, oracle):
    """BASELINE config: 100k dirty leaves into the 16^6-leaf trie; root equals the oracle's full recompute."""
    depth, n = 6, 100_000
    t = ctx.trie_open(depth)
    o = oracle.ctrie(depth)
    assert t.root() == o.root()
    rng = np.random.default_rng(1)
    pos = rng.choice(16 ** depth, size=n, replace=False).astype(np.uint32)
    keys = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    keys[:, 0] = (pos >> 16) & 0xff
    keys[:, 1] = (pos >> 8) & 0xff
    keys[:, 2] = pos & 0xff
    vals = [rng.integers(0, 256, 78, dtype=np.uint8).tobytes() for _ in range(n)]
    v, voff = oracle_lib.csr(vals, np.uint32)
    flat = np.ascontiguousarray(keys.reshape(-1))
    assert t.update(flat, v, voff, n) == o.update(flat, vals)
    t.close()


def test_fuzz_many_tries_one_forest(ctx, oracle):
    """400 random tries (prefix-heavy keys, empty / tiny / large values, empty and single-key tries) built as ONE forest by
    phant_gpu_mpt_roots and each compared with the oracle; covers both arena layouts (prefix keys force the general one)."""
    rng = np.random.default_rng(99)
    for prefixy in (True, False):
        lists = []
        for _ in range(200):
            n = int(rng.choice([0, 1, 2, 3, 7, 20, 60, 150]))
            if prefixy:
                kv = random_prefixy_items(rng, n) if n else []
            else:
                keys = sorted({rng.integers(0, 256, 8, dtype=np.uint8).tobytes() for _ in range(n)})
                kv = [(k, rng.integers(0, 256, int(rng.choice([0, 1, 31, 32, 33, 200, 700])), dtype=np.uint8).tobytes()) for k in keys]
            lists.append(kv)
        flat = [x for l in lists for x in l]
        keys, koff = oracle_lib.csr([k for k, _ in flat], np.uint32)
        vals, voff = oracle_lib.csr([v for _, v in flat], np.uint64)
        seg = np.zeros(len(lists) + 1, np.uint32)
        seg[1:] = np.cumsum([len(l) for l in lists])
        got = ctx.mpt_roots(keys, koff, vals, voff, seg, len(lists))
        for i, kv in enumerate(lists):
            assert got[i] == oracle.mptize(kv), (prefixy, i, len(kv))


# ---------------------------------------------------------------------------------------------------------------
# U kind 1: sparse resident secure trie (dense top + sparse buckets), checked against a full recompute by the oracle
# ---------------------------------------------------------------------------------------------------------------
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


def test_sparse_resident_trie_grows_updates_and_shrinks(ctx, oracle):
    """inserts across the dense-depth thresholds (L = 0 -> 1 -> 2 -> 3), value updates (no merge), deletes (incl. keys that
    are not there), mixed batches; after every update the root equals oracle.mptize over the whole key set"""
    rng = np.random.default_rng(5)
    trie = ctx.trie_open(0, kind=1)
    state = {}
    assert trie.root() == oracle.mptize([])

    def rkey():
        return rng.integers(0, 256, 32, dtype=np.uint8).tobytes()

    def rval():
        return rng.integers(0, 256, int(rng.integers(1, 120)), dtype=np.uint8).tobytes()

    def check(root):
        assert root == oracle.mptize(sorted(state.items())), len(state)
        assert trie.root() == root

    check(_apply(trie, state, {rkey(): rval() for _ in range(7)}))
    check(_apply(trie, state, {rkey(): rval() for _ in range(150)}))
    check(_apply(trie, state, {rkey(): rval() for _ in range(400)}))          # crosses 256: L = 1
    some = list(state)[:60]
    check(_apply(trie, state, {k: rval() for k in some}))                     # pure value updates
    check(_apply(trie, state, {rkey(): rval() for _ in range(6000)}))         # crosses 4096: L = 2
    mixed = {k: b"" for k in list(state)[100:400]}                            # deletes ...
    mixed.update({rkey(): rval() for _ in range(200)})                        # ... inserts ...
    mixed.update({k: rval() for k in list(state)[1000:1300]})                 # ... replacements ...
    mixed.update({rkey(): b"" for _ in range(20)})                            # ... and deletes of absent keys, in one batch
    check(_apply(trie, state, mixed))
    check(_apply(trie, state, {rkey(): rval() for _ in range(70000)}))        # crosses 65536: L = 3
    check(_apply(trie, state, {k: rval() for k in list(state)[::97]}))
    check(_apply(trie, state, {k: b"" for k in list(state)[: len(state) - 3000]}))  # shrink far below the bound: L drops
    check(_apply(trie, state, {k: b"" for k in list(state)}))                 # everything gone: the empty root
    assert trie.root() == oracle.mptize([])
    check(_apply(trie, state, {rkey(): rval() for _ in range(30)}))
    trie.close()


def test_sparse_resident_trie_keeps_mptize_rules_when_keys_are_not_uniform(ctx, oracle):
    """keys that share long prefixes (extensions above the buckets, single-child dense nodes): the dense-top premise fails,
    the structure must notice on the device and fall back to fewer dense levels; values < 32 bytes give embedded leaves"""
    rng = np.random.default_rng(6)
    trie = ctx.trie_open(0, kind=1)
    state = {}
    base = rng.integers(0, 256, 32, dtype=np.uint8)
    changes = {}
    for i in range(700):                                     # > 256 keys, all under ONE top nibble and a 5-byte shared prefix
        k = base.copy()
        k[5:] = rng.integers(0, 256, 27, dtype=np.uint8)
        changes[k.tobytes()] = rng.integers(0, 256, int(rng.integers(1, 40)), dtype=np.uint8).tobytes()
    assert _apply(trie, state, changes) == oracle.mptize(sorted(state.items()))
    more = {}
    for i in range(300):                                     # pairs differing only in the last nibble: deep embedded leaves
        k = rng.integers(0, 256, 32, dtype=np.uint8)
        for last in (0x10, 0x11):
            k2 = k.copy(); k2[31] = last
            more[k2.tobytes()] = bytes([1 + i % 100])
    assert _apply(trie, state, more) == oracle.mptize(sorted(state.items()))
    assert _apply(trie, state, {k: b"" for k in list(changes)[:650]}) == oracle.mptize(sorted(state.items()))
    trie.close()


def test_sparse_resident_trie_refuses_bad_updates(ctx, oracle):
    """a repeated key and device pointers are refused; the root stays what it was and the next update is right, on an empty
    trie and on one that holds keys"""
    from phant_b200 import gpu
    trie = ctx.trie_open(0, kind=1)
    k = np.arange(64, dtype=np.uint8)
    k[32:] = k[:32]                                           # the same key twice
    with pytest.raises(gpu.PhantGpuError) as e:
        trie.update(k, np.array([1, 2], np.uint8), np.array([0, 1, 2], np.uint32), 2)
    assert e.value.code == -1
    assert trie.root() == oracle.mptize([])
    ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
    with pytest.raises(gpu.PhantGpuError):
        trie.update(k[:32], np.array([1], np.uint8), np.array([0, 1], np.uint32), 1)
    ctx.set_flags(0)
    assert trie.root() == oracle.mptize([])
    rng = np.random.default_rng(8)
    state = {}
    keys = [rng.integers(0, 256, 32, dtype=np.uint8).tobytes() for _ in range(600)]
    root = _apply(trie, state, {x: rng.integers(0, 256, 70, dtype=np.uint8).tobytes() for x in keys[:500]})
    assert root == oracle.mptize(sorted(state.items()))
    for dup in (keys[3], keys[550]):                          # a key already held, and a new one, each twice in one batch
        bad = keys[400:450] + [dup, dup]
        kk = np.frombuffer(b"".join(bad), np.uint8)
        v, voff = oracle_lib.csr([bytes([i % 200 + 1]) * 40 for i in range(len(bad))], np.uint32)
        with pytest.raises(gpu.PhantGpuError) as e:
            trie.update(kk, v, voff, len(bad))
        assert e.value.code == -1
        assert trie.root() == root
    changes = {x: b"" for x in keys[:50]}
    changes.update({x: rng.integers(0, 256, 90, dtype=np.uint8).tobytes() for x in keys[450:]})
    assert _apply(trie, state, changes) == oracle.mptize(sorted(state.items()))
    trie.close()


def test_fixture_post_state_roots_by_updating_the_pre_state_trie(ctx, oracle, golden):
    """the StateDB.root() hook as a resident structure (blockchain.zig:83-85): for each of the 84 fixture tests, load the `pre`
    accounts into a sparse resident trie (root must be genesisBlockHeader.stateRoot), then apply ONLY the accounts the block(s)
    changed / created / destroyed and require the last valid block's stateRoot -- both expectations are the fixture's"""
    from helpers import secure_account_items
    g = golden("fixture_states.json.gz")
    done = 0
    for t in g["tests"]:
        pre = dict(secure_account_items(oracle.keccak256, oracle.mptize, g["tables"][t["pre"]]))
        post = dict(secure_account_items(oracle.keccak256, oracle.mptize, g["tables"][t["post"]]))
        trie = ctx.trie_open(0, kind=1)
        state = {}
        if pre:
            assert _apply(trie, state, pre).hex() == t["pre_root"], t["name"]
        changes = {k: v for k, v in post.items() if pre.get(k) != v}
        changes.update({k: b"" for k in pre if k not in post})
        root = _apply(trie, state, changes) if changes else trie.root()
        assert root.hex() == t["post_root"], t["name"]
        trie.close()
        done += 1
    assert done == 84
