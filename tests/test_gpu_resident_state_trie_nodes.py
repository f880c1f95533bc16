"""Trie nodes by path from the resident world state (phant_gpu_resident_state_trie_nodes, snap's GetTrieNodes): every answer
equals the CPU statement (tests/trie_node_model.py) -- status 1 with the node's RLP exactly where the account trie or the named
storage trie holds the root or a node of 32 bytes or more starting at that path, status 2 everywhere else -- in the caller's
order, and the state is left exactly as it was.  A full heal from the empty path, level by level, fetches exactly the
statement's node set, and W (phant_gpu_verify_witness) proves every account from it."""
import numpy as np
import pytest

from helpers import _rlp_item
from phant_b200 import gpu
from phant_b200 import host
from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel, change_diff, hashed_table, load_diff
from test_gpu_resident_state import block, grow_account, rkey, rval, u32be
from test_gpu_resident_state_witness import fixture_touched
from test_gpu_transition_roots_at_size import build_state
from trie_node_model import nibbles, pack, probe_paths, state_nodes

pytestmark = pytest.mark.gpu

EMPTY = host.EMPTY_MPT_ROOT


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


def ask(st, items):
    """items: [(storage account key or None for the account trie, nibble path)] -> (status, [bytes])"""
    owners = list(dict.fromkeys(o for o, _ in items if o is not None))
    oi = {o: i for i, o in enumerate(owners)}
    packed = [pack(p) for _, p in items]
    paths = np.frombuffer(b"".join(b for b, _ in packed), np.uint8).copy() if items else np.zeros(0, np.uint8)
    lens = np.array([n for _, n in packed], np.uint8)
    tries = np.array([0 if o is None else 1 + oi[o] for o, _ in items], np.uint32)
    sa = np.frombuffer(b"".join(owners), np.uint8).copy() if owners else None
    return st.trie_nodes(paths, lens, tries, sa)


def checked(oracle, st, m, items, want=None):
    """ask, and compare every answer with the statement; the state is unchanged"""
    want = state_nodes(oracle.keccak256, m) if want is None else want
    root, info = st.root(), st.info()
    status, blobs = ask(st, items)
    assert st.root() == root
    assert {k: v for k, v in st.info().items() if k != "device_bytes"} == {k: v for k, v in info.items() if k != "device_bytes"}
    assert len(status) == len(blobs) == len(items)
    for (o, p), s, b in zip(items, status, blobs):
        w = want.get((o, p))
        assert (int(s), b) == ((1, w) if w is not None else (2, b"")), (o.hex() if o else None, p)
    return status, blobs


def around(m, rng, owners_sample=None, diverge=True):
    """probe paths of the account trie and of the storage tries of `owners_sample` (default: all accounts with storage)"""
    items = [(None, p) for p in probe_paths(m.acc, rng, diverge)]
    for k in (owners_sample if owners_sample is not None else [k for k, a in m.acc.items() if a.storage]):
        a = m.acc.get(k)
        items += [(k, p) for p in probe_paths(a.storage if a else [], rng, diverge)]
    return items


def test_fixtures(ctx, oracle, golden):
    g = golden("fixture_states.json.gz")
    rng = np.random.default_rng(41)
    n = 0
    for t in g["tests"]:
        pre = hashed_table(oracle.keccak256, g["tables"][t["pre"]])
        st = ctx.resident_state()
        m = StateModel(oracle)
        st.apply(**load_diff(pre).arrays())
        m.apply(load_diff(pre))
        want = state_nodes(oracle.keccak256, m)
        items = list(want) + around(m, rng)
        bare = [k for k, a in m.acc.items() if not a.storage]
        ghost = rkey(rng)
        items += [(k, ()) for k in bare[:3]] + [(ghost, ()), (ghost, (1, 2))]
        items.append(items[0])  # a repeat
        rng.shuffle(items)
        status, blobs = checked(oracle, st, m, items, want)
        assert set(want) <= {it for it, s in zip(items, status) if s == 1}
        d = change_diff(pre, hashed_table(oracle.keccak256, g["tables"][t["post"]]))
        assert st.apply(**d.arrays()).hex() == t["post_root"], t["name"]
        st.close()
        n += 1
    assert n == 84


def _items(node):
    """the top-level items of a node: [(is_list, raw item bytes, payload)]"""
    top = _rlp_item(node, 0, len(node))
    out, pos = [], top[1]
    while pos < top[2]:
        it = _rlp_item(node, pos, top[2])
        out.append((it[0], node[pos:it[3]], node[it[1]:it[2]]))
        pos = it[3]
    return out


def _hp(b):
    nib = [x for c in b for x in (c >> 4, c & 15)]
    return b[0] >> 4 >= 2, tuple(nib[1:] if b[0] >> 4 & 1 else nib[2:])


def children(o, p, node):
    """what a healer asks for next below node (trie o, path p): (trie, path, reference) of every child referenced by hash,
    and at an account leaf its storage root"""
    its = _items(node)
    out = []

    def child(path, it):
        if it[0]:
            out.extend(children(o, path, it[1]))  # embedded: walked in place
        elif len(it[2]) == 32:
            out.append((o, path, it[2]))

    if len(its) == 17:
        for c in range(16):
            child(p + (c,), its[c])
        return out
    leaf, nib = _hp(its[0][2])
    if not leaf:
        child(p + nib, its[1])
    elif o is None:
        full = p + nib
        sroot = _items(its[1][2])[2][2]
        if sroot != EMPTY:
            out.append((bytes(full[i] << 4 | full[i + 1] for i in range(0, 64, 2)), (), sroot))
    return out


def heal(oracle, st):
    """a trie-node sync from the state root: level by level, every child referenced by hash of what was fetched, each
    checked against the reference its parent holds"""
    got, frontier = {}, [(None, (), st.root())]
    while frontier:
        status, blobs = ask(st, [(o, p) for o, p, _ in frontier])
        nxt = []
        for (o, p, ref), s, b in zip(frontier, status, blobs):
            assert s == 1 and oracle.keccak256(b) == ref, (o, p)
            got[(o, p)] = b
            nxt += children(o, p, b)
        frontier = nxt
    return got


def healed_checked(ctx, oracle, st, m):
    got = heal(oracle, st)
    assert got == state_nodes(oracle.keccak256, m)
    nodes = sorted(set(got.values()))
    off = np.zeros(len(nodes) + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in nodes])
    keys = sorted(m.acc)
    n = len(keys)
    bitmap, status = np.zeros((n + 63) // 64, np.uint64), np.zeros(n, np.uint8)
    voff, vlen = np.zeros(n, np.uint64), np.zeros(n, np.uint32)
    data = np.frombuffer(b"".join(nodes) + bytes(64), np.uint8).copy()
    ctx.verify_witness(len(nodes), data, off, n, np.frombuffer(b"".join(keys), np.uint8).copy(), np.frombuffer(st.root(), np.uint8).copy(),
                       1, bitmap, status, voff, vlen, nodes_bytes=int(off[-1]))
    assert (status == 1).all()
    for i, k in enumerate(keys):
        assert data[int(voff[i]):int(voff[i]) + int(vlen[i])].tobytes() == m.leaf(k)
    return got


def test_heal_block_sequence(ctx, oracle):
    rng = np.random.default_rng(23)
    st = ctx.resident_state()
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(20000)]
    big, doomed, reborn = keys[0], keys[1], keys[2]
    fields = lambda: (int(rng.integers(0, 1 << 20)), u32be(rng.integers(0, 1 << 60)), rkey(rng))  # noqa: E731
    writes = [(k, rkey(rng), rval(rng)) for k in keys[3:1003] for _ in range(int(rng.integers(1, 30)))]
    writes += grow_account(rng, m, doomed, 5000) + grow_account(rng, m, reborn, 300)
    d = block(rng, m, {k: fields() for k in keys}, writes)
    st.apply(**d.arrays())
    m.apply(d)
    healed_checked(ctx, oracle, st, m)
    for target in (1000, 70000, 200, 0):  # `big`: L 0 -> 1 -> 3 -> 0, then no storage
        touched = {keys[i]: fields() for i in rng.choice(np.arange(3, 20000), 40, replace=False)}
        w = grow_account(rng, m, big, target)
        small = [keys[i] for i in rng.choice(np.arange(3, 1003), 40, replace=False)]
        w += [(k, sk, ZERO32) for k in small[:20] for sk in list(m.acc[k].storage)[:2]]
        w += [(k, rkey(rng), rval(rng)) for k in small[20:]]
        d = block(rng, m, touched, w)
        st.apply(**d.arrays())
        m.apply(d)
        if target == 70000:
            healed_checked(ctx, oracle, st, m)
        else:
            checked(oracle, st, m, around(m, rng, [big, doomed, reborn], diverge=False)[::7])
    gone = sorted(keys[3000:3400])[100:110]
    d = block(rng, m, {doomed: (0, ZERO32, ZERO32), reborn: fields(), **{k: (0, ZERO32, ZERO32) for k in gone}},
              [(reborn, rkey(rng), rval(rng)) for _ in range(40)], flags={doomed: DELETE, reborn: CLEAR, **{k: DELETE for k in gone}})
    st.apply(**d.arrays())
    m.apply(d)
    got = healed_checked(ctx, oracle, st, m)
    assert not any(o == doomed for o, _ in got)
    checked(oracle, st, m, [(doomed, ()), (big, ()), (reborn, ())] + [(k, ()) for k in gone])
    st.close()


def test_crafted_keys(ctx, oracle):
    rng = np.random.default_rng(7)
    st = ctx.resident_state()
    m = StateModel(oracle)
    a, b, c, e = rkey(rng), rkey(rng), rkey(rng), rkey(rng)
    one = lambda: bytes([int(rng.integers(1, 0x80))]).rjust(32, b"\x00")  # noqa: E731
    ka = [bytes([0xa0 | int(rng.integers(0, 16))]) + rkey(rng)[1:] for _ in range(300)]  # breaks the dense-top premise
    kb = [bytes([int(rng.integers(0, 15)) << 4 | int(rng.integers(0, 16))]) + rkey(rng)[1:] for _ in range(600)]  # no nibble f on top
    kc = []
    for i in range(150):  # pairs sharing 62 nibbles with 1-byte values: leaves embedded in their branch
        base = b"\x77" * 28 + bytes([i]) + rkey(rng)[:2]
        kc += [base + bytes([0x10]), base + bytes([0x11])]
    deep = []
    for i in range(20):  # pairs sharing 63 nibbles with full values: hashed leaves at depth 64
        base = rkey(rng)[:31] + bytes([0x40 | (i & 15)])
        deep += [base[:31] + bytes([0x50]), base[:31] + bytes([0x51])]
    w = [(a, k, one()) for k in ka] + [(b, k, one()) for k in kb] + [(c, k, one()) for k in kc] + [(e, k, b"\xff" + rkey(rng)[1:]) for k in deep]
    d = block(rng, m, {a: (1, u32be(1), ZERO32), b: (2, u32be(2), ZERO32), c: (3, u32be(3), ZERO32), e: (4, u32be(4), ZERO32),
                       **{k: (1, u32be(1), ZERO32) for k in [rkey(rng) for _ in range(400)]}}, w)
    st.apply(**d.arrays())
    m.apply(d)
    want = state_nodes(oracle.keccak256, m)
    assert sum(1 for o, p in want if o == e and len(p) == 64) == 40
    items = around(m, rng, [a, b, c, e])
    items += [(b, (15,)), (b, (15, 3)), (b, (15, 0, 0))]  # under the dense top's empty child
    checked(oracle, st, m, items, want)
    st.close()


def test_empty_state(ctx, oracle):
    rng = np.random.default_rng(8)
    st = ctx.resident_state()
    m = StateModel(oracle)
    k = rkey(rng)
    status, blobs = checked(oracle, st, m, [(None, ()), (None, nibbles(k)), (None, (3,)), (k, ()), (k, nibbles(k)[:7])])
    assert (status == 2).all()
    status, blobs = st.trie_nodes(np.zeros(0, np.uint8), np.zeros(0, np.uint8))
    assert len(status) == 0 and blobs == []
    st.close()


def test_after_revert(ctx, oracle):
    rng = np.random.default_rng(10)
    st = ctx.resident_state()
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(2000)]
    d = block(rng, m, {k: (1, u32be(5), ZERO32) for k in keys}, [(k, rkey(rng), rval(rng)) for k in keys[:300] for _ in range(8)])
    st.apply(**d.arrays())
    m.apply(d)
    st.set_journal(4)
    models = [m.copy()]
    for i in range(3):
        touched = {keys[int(j)]: (2, u32be(i + 7), ZERO32) for j in rng.choice(2000, 60, replace=False)}
        w = [(k, list(m.acc[k].storage)[0], ZERO32) for k in keys[i * 30:i * 30 + 30]] + [(k, rkey(rng), rval(rng)) for k in keys[500:520]]
        touched[keys[1500 + i]] = (0, ZERO32, ZERO32)
        d = block(rng, m, touched, w, flags={keys[1500 + i]: DELETE})
        st.apply(**d.arrays())
        m.apply(d)
        models.append(m.copy())
    assert st.revert(2) == models[1].root()
    healed_checked(ctx, oracle, st, models[1])
    checked(oracle, st, models[1], around(models[1], rng, keys[:40] + keys[1500:1503], diverge=False)[::3])
    st.close()


def test_refusals_and_one_result(ctx, oracle):
    rng = np.random.default_rng(9)
    st = ctx.resident_state()
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(300)]
    d = block(rng, m, {k: (1, u32be(5), ZERO32) for k in keys}, [(k, rkey(rng), rval(rng)) for k in keys[:50] for _ in range(4)])
    st.apply(**d.arrays())
    m.apply(d)
    st.set_journal(2)
    root, info = st.root(), st.info()
    k1 = keys[0]
    p2 = np.zeros(64, np.uint8)
    l2 = np.array([0, 3], np.uint8)
    t2 = np.array([0, 1], np.uint32)
    a1 = np.frombuffer(k1, np.uint8).copy()
    a2 = np.frombuffer(k1 + k1, np.uint8).copy()
    l65, t_2 = np.array([0, 65], np.uint8), np.array([0, 2], np.uint32)  # kept alive: the requests hold raw pointers
    Q = gpu.TrieNodeRequest
    bad = [Q(2, None, l2.ctypes.data, None, 0, None),                                  # NULL paths
           Q(2, p2.ctypes.data, None, None, 0, None),                                  # NULL lengths
           Q(2, p2.ctypes.data, l65.ctypes.data, None, 0, None),  # a path of 65 nibbles
           Q(2, p2.ctypes.data, l2.ctypes.data, t_2.ctypes.data, 1, a1.ctypes.data),  # no storage account 2
           Q(2, p2.ctypes.data, l2.ctypes.data, t2.ctypes.data, 1, None),               # NULL storage accounts
           Q(2, p2.ctypes.data, l2.ctypes.data, t2.ctypes.data, 2, a2.ctypes.data),    # the same storage account twice
           Q((1 << 28) + 1, p2.ctypes.data, l2.ctypes.data, None, 0, None)]            # too many paths
    import torch
    dp = torch.zeros(64, dtype=torch.uint8, device="cuda")
    bad.append(Q(2, dp.data_ptr(), l2.ctypes.data, None, 0, None))                      # device pointers
    hs, ho, hn = np.zeros(2, np.uint8), np.zeros(3, np.uint64), np.zeros(1 << 16, np.uint8)
    held = gpu.TrieNodes(hs.ctypes.data, ho.ctypes.data, hn.ctypes.data)
    for q in bad:
        assert st.trie_nodes_raw(q)[0] == -1
        assert st.trie_nodes_copy_raw(held) == -1  # nothing held
    # storage_account32 may be NULL when no path names a storage trie
    assert st.trie_nodes_raw(Q(2, p2.ctypes.data, l2.ctypes.data, None, 5, None))[0] == 0
    assert st.root() == root and st.info()["journal_applies"] == info["journal_applies"]
    good = gpu.ResidentState._trie_node_request(p2, l2, t2, a1)
    rc, size = st.trie_nodes_raw(good)
    assert rc == 0 and size.n_nodes >= 1
    proofs = gpu.Proofs(*([None] * 11))
    assert st.prove_copy_raw(proofs) == -1 and st.witness_copy_raw(np.zeros(1 << 16, np.uint8), np.zeros(1 << 12, np.uint64)) == -1
    # read, range and codes keep it; the result counts in device_bytes while held
    assert st.trie_nodes_raw(good)[0] == 0
    st.read(a1)
    st.range([(bytes(32), b"\xff" * 32, 4)])
    st.codes(np.zeros(32, np.uint8))
    held_bytes = st.info()["device_bytes"]
    status, off = np.zeros(2, np.uint8), np.zeros(3, np.uint64)
    nodes = np.zeros(max(size.nodes_bytes, 1), np.uint8)
    assert st.trie_nodes_copy_raw(gpu.TrieNodes(status.ctypes.data, off.ctypes.data, nodes.ctypes.data)) == 0
    assert st.info()["device_bytes"] < held_bytes
    assert list(status) == [1, 2] or list(status) == [1, 1]
    assert oracle.keccak256(nodes[:int(off[1])].tobytes()) == root
    # trie nodes drop a held proof result, and every later call of another kind drops trie nodes
    assert st.prove_raw(gpu.ResidentState._request(a1))[0] == 0
    assert st.trie_nodes_raw(good)[0] == 0
    assert st.prove_copy_raw(proofs) == -1
    rc, _ = st.witness_raw(gpu.ResidentState._diff(**Diff([(k1, 0, 1, u32be(1), ZERO32)]).arrays()))
    assert rc == 0 and st.trie_nodes_copy_raw(held) == -1
    for after in (lambda: st.prove(a1), lambda: st.set_journal(2), lambda: st.apply(**Diff([(k1, 0, 2, u32be(2), ZERO32)]).arrays()),
                  lambda: st.revert(1)):
        assert st.trie_nodes_raw(good)[0] == 0
        after()
        assert st.trie_nodes_copy_raw(held) == -1
    st.close()


def test_at_size(ctx, oracle):
    """100k accounts, 1M slots: a heal-shaped request of existing and missing paths matches the statement on the account trie
    and on the storage tries it names; launches follow trie depths, not the request's size; H2D is about the request"""
    rng = np.random.default_rng(103)
    m, full = build_state(oracle, rng, 100_000, [(i * 100, 1000) for i in range(1000)])
    st = ctx.resident_state()
    assert st.apply(**full.arrays()) == m.root()
    from trie_node_model import served, storage_value, trie_nodes
    _, acc = trie_nodes(oracle.keccak256, {k: m.leaf(k) for k in m.acc})
    want = {(None, p): e for p, e in served(acc).items()}
    rich = [k for k, a in m.acc.items() if a.storage]
    owners = [rich[int(i)] for i in rng.choice(len(rich), 64, replace=False)]
    for k in owners:
        _, sn = trie_nodes(oracle.keccak256, {sk: storage_value(v) for sk, v in m.acc[k].storage.items()})
        want.update(((k, p), e) for p, e in served(sn).items())
    have_acc = [p for o, p in want if o is None and len(p) <= 8]
    have_st = [(o, p) for o, p in want if o is not None]
    items = [(None, have_acc[int(i)]) for i in rng.choice(len(have_acc), 600, replace=False)]
    items += [have_st[int(i)] for i in rng.choice(len(have_st), 320, replace=False)]
    items += [(None, tuple(int(x) for x in rng.integers(0, 16, int(rng.integers(1, 9))))) for _ in range(52)]
    items += [(owners[int(rng.integers(0, 64))], tuple(int(x) for x in rng.integers(0, 16, int(rng.integers(1, 6))))) for _ in range(52)]
    checked(oracle, st, m, items, want)
    launches = []
    for n in (10, 2000):
        sel = [have_acc[int(i) % len(have_acc)] for i in range(n)]
        ctx.reset_stats()
        ask(st, [(None, p) for p in sel])
        s = ctx.stats()
        launches.append(s["launches"])
        assert s["h2d_bytes"] <= 37 * n + 4096, s
    assert launches[1] < 2 * launches[0], launches
    st.close()


def compact(path):
    """a nibble path, compact-encoded as a healer sends it (flag nibble 0 even / 1 odd)"""
    nib = list(path)
    head = bytes([0x10 | nib[0]]) if len(nib) & 1 else b"\x00"
    rest = nib[1:] if len(nib) & 1 else nib
    return head + bytes(rest[i] << 4 | rest[i + 1] for i in range(0, len(rest), 2))


def test_host_layer(ctx, oracle, golden):
    """host.ResidentStateDB.get_trie_nodes on every fixture: a heal through snap's wire pathsets (compact paths, storage sets
    led by the account hash) fetches exactly the statement's nodes; bad encodings give b"", max_bytes cuts the answer after
    the blob that crosses it, and a root other than the current one gives []"""
    g = golden("fixture_states.json.gz")
    for t in g["tests"]:
        old, _, _ = fixture_touched(g["tables"][t["pre"]], g["tables"][t["post"]])
        rs = host.ResidentStateDB(ctx)
        if old:
            assert rs.apply(old).hex() == t["pre_root"], t["name"]
        root = rs.state.root()
        m = StateModel(oracle)
        m.apply(load_diff(hashed_table(oracle.keccak256, g["tables"][t["pre"]])))
        want = state_nodes(oracle.keccak256, m)
        got, frontier = {}, [(None, (), root)]
        while frontier:
            sets, order = [], []
            for o, p, ref in frontier:  # one pathset per account trie node, one per storage trie with all its paths
                if o is None:
                    sets.append([compact(p)])
                    order.append((o, p, ref))
            by = {}
            for o, p, ref in frontier:
                if o is not None:
                    by.setdefault(o, []).append((p, ref))
            for o, ps in by.items():
                sets.append([o] + [compact(p) for p, _ in ps])
                order += [(o, p, ref) for p, ref in ps]
            blobs = rs.get_trie_nodes(root, sets, max_bytes=1 << 30)
            assert len(blobs) == len(order)
            nxt = []
            for (o, p, ref), b in zip(order, blobs):
                assert oracle.keccak256(b) == ref
                got[(o, p)] = b
                nxt += children(o, p, b)
            frontier = nxt
        assert got == want, t["name"]
        if want:
            sets = [[b""], [b"\x20"], [b"\x3a"], [b"\x05"], [b"\x00" * 34], [compact(())], [b"\x11"]]
            blobs = rs.get_trie_nodes(root, sets)
            assert blobs[:5] == [b""] * 5 and blobs[5] == want[(None, ())]
            assert blobs[6] == want.get((None, (1,)), b"")
            paths = [[compact(p)] for o, p in want if o is None] * 3
            full = rs.get_trie_nodes(root, paths, max_bytes=1 << 30)
            cut = len(want[(None, ())]) + 1
            part = rs.get_trie_nodes(root, paths, max_bytes=cut)
            total, n = 0, 0
            for b in full:
                total, n = total + len(b), n + 1
                if total > cut:
                    break
            assert part == full[:n] and n < len(full)
            assert rs.get_trie_nodes(b"\x01" * 32, paths) == []
        rs.close()
