"""Forks of the resident world state (phant_gpu_resident_state_fork) on the GPU: a fork holds exactly the state revert(back)
would return to -- root, counts, storage roots, reads, dumps, proofs, trie nodes and witnesses all equal those of a twin that
really reverted, or of the model at that root -- while the parent is not changed at all (root, info, journal, a held result).
The fork is independent of its parent (either may move, be closed first, or be forked again), snap's boundary proofs and
trie nodes are served at a pivot through host.ResidentStateDB.fork_at, and the costs stay within a device-to-device copy
plus `back` replays."""
import ctypes as C

import numpy as np
import pytest

from phant_b200 import gpu
from phant_b200 import host
from resident_state_model import CLEAR, DELETE, ZERO32, StateModel, change_diff, hashed_table, load_diff
from test_gpu_resident_state import apply_checked, block, grow_account, rkey, rval, u32be
from test_gpu_resident_state_proofs import proofs_checked, request_for
from test_gpu_resident_state_trie_nodes import around, checked, healed_checked
from test_gpu_transition_roots_at_size import block_diff, build_state
from trie_node_model import state_nodes

pytestmark = pytest.mark.gpu

E_INVALID = -1
EMPTY = host.EMPTY_MPT_ROOT


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


def counts(m):
    return len(m.acc), sum(len(a.storage) for a in m.acc.values())


def db_over(ctx, st):
    """a host.ResidentStateDB over the gpu.ResidentState st (not owned: closing st stays the caller's)"""
    db = host.ResidentStateDB.__new__(host.ResidentStateDB)
    db.ctx, db.state, db.code_state, db.journal = ctx, st, st, 0
    return db


def reads_checked(st, m, akeys, slots):
    """read() of accounts akeys and slots [(account index, slot key)] on st equals model m"""
    sa = np.array([i for i, _ in slots], np.uint32) if slots else None
    sk = np.frombuffer(b"".join(k for _, k in slots), np.uint8).copy() if slots else None
    r, root = st.read(np.frombuffer(b"".join(akeys), np.uint8).copy(), sa, sk)
    assert root == (m.root() if m.acc else EMPTY)
    for i, k in enumerate(akeys):
        a = m.acc.get(k)
        if a is None:
            assert r["account_status"][i] == 2
            continue
        assert r["account_status"][i] == 1 and int(r["nonce"][i]) == a.nonce
        assert r["balance32"][i].tobytes() == a.balance and r["code_hash32"][i].tobytes() == a.code_hash
        assert r["storage_root32"][i].tobytes() == m.storage_root(k)
    for j, (i, k) in enumerate(slots):
        a = m.acc.get(akeys[i])
        v = a.storage.get(k) if a else None
        assert r["slot_status"][j] == (1 if v else 2) and r["slot_vals32"][j].tobytes() == (v or ZERO32)


def test_fixtures(ctx, oracle, golden):
    """every fixture: fork(1) after the change diff is the pre-state, fork(0) the post-state -- root, counts, reads and proofs"""
    g = golden("fixture_states.json.gz")
    rng = np.random.default_rng(61)
    n = 0
    for t in g["tests"]:
        pre, post = hashed_table(oracle.keccak256, g["tables"][t["pre"]]), hashed_table(oracle.keccak256, g["tables"][t["post"]])
        st = ctx.resident_state()
        st.set_journal(1)
        before = StateModel(oracle)
        apply_checked(st, before, load_diff(pre))
        after = before.copy()
        d = change_diff(pre, post)
        assert apply_checked(st, after, d).hex() == t["post_root"], t["name"]
        for back, m, root in ((1, before, t["pre_root"]), (0, after, t["post_root"])):
            f = st.fork(back)
            assert f.root().hex() == root, (t["name"], back)
            info = f.info()
            assert (info["n_accounts"], info["n_slots"]) == counts(m) and info["journal_applies"] == 0
            other = after if m is before else before
            akeys, slots = request_for(rng, m, list(m.acc) + [k for k in other.acc if k not in m.acc])
            reads_checked(f, m, akeys, slots)
            proofs_checked(ctx, oracle, f, m, akeys, slots)
            f.close()
        assert st.root().hex() == t["post_root"] and st.info()["journal_applies"] == 1
        st.close()
        n += 1
    assert n == 84


def sequence(ctx, oracle, rng, states):
    """the revert tests' 9 blocks (an account going L 0 -> 3 and back, accounts destroyed holding 5,000 slots and re-created,
    an empty block) applied to every state of `states` at journal depth 16.  Returns (hist, diffs, keys): hist[i] = (model,
    root) after i blocks."""
    for st in states:
        st.set_journal(16)
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(6000)]
    big, doomed, reborn = keys[0], keys[1], keys[2]
    fields = lambda: (int(rng.integers(0, 1 << 20)), u32be(rng.integers(0, 1 << 60)), rkey(rng))  # noqa: E731
    hist, diffs = [(m.copy(), EMPTY)], []

    def step(d):
        diffs.append(d)
        root = apply_checked(states[0], m, d)
        for st in states[1:]:
            assert st.apply(**d.arrays()) == root
        hist.append((m.copy(), root))

    writes = [(k, rkey(rng), rval(rng)) for k in keys[3:1003] for _ in range(int(rng.integers(1, 10)))]
    writes += grow_account(rng, m, big, 200) + grow_account(rng, m, doomed, 5000) + grow_account(rng, m, reborn, 300)
    step(block(rng, m, {k: fields() for k in keys}, writes))
    for target in (1000, 5000, 70000, 5000, 1000, 200):
        touched = {keys[i]: fields() for i in rng.choice(np.arange(3, 6000), 30, replace=False)}
        w = grow_account(rng, m, big, target)
        small = [keys[i] for i in rng.choice(np.arange(3, 1003), 30, replace=False)]
        w += [(k, list(m.acc[k].storage)[0], rval(rng)) for k in small if m.acc[k].storage]
        w += [(k, rkey(rng), ZERO32) for k in small[:5]]
        step(block(rng, m, touched, w))
    step(block(rng, m, {doomed: (0, ZERO32, ZERO32), reborn: fields()}, [(reborn, rkey(rng), rval(rng)) for _ in range(40)],
               flags={doomed: DELETE, reborn: CLEAR}))
    step(block(rng, m, {}, []))
    return hist, diffs, keys


def test_block_sequence_at_every_back(ctx, oracle):
    """for every back 0..9, fork(back) against a twin that ran revert(back): root, counts, storage roots, the dump (equal to
    the parent's past-root dump), trie nodes against the statement, proofs through V at read(back)'s root, and the next
    block's witness (byte-equal to the twin's, and through T the root the parent recorded)"""
    rng = np.random.default_rng(71)
    st, twin = ctx.resident_state(), ctx.resident_state()
    hist, diffs, keys = sequence(ctx, oracle, rng, [st, twin])
    big, doomed, reborn = keys[:3]
    nb = len(diffs)
    assert nb == 9 and st.info()["journal_applies"] == 9
    for back in range(nb + 1):
        if back:
            assert twin.revert(1) == hist[nb - back][1]
        m, root = hist[nb - back]
        root0, info0 = st.root(), st.info()
        f = st.fork(back)
        assert st.root() == root0 and st.info() == info0
        assert f.root() == twin.root() == root == st.read(np.zeros(0, np.uint8), back=back)[1]
        fi, ti = f.info(), twin.info()
        assert (fi["n_accounts"], fi["n_slots"]) == (ti["n_accounts"], ti["n_slots"]) == counts(m)
        ak = np.frombuffer(b"".join(keys[:600] + [rkey(rng)]), np.uint8).copy()
        assert np.array_equal(f.read(ak)[0]["storage_root32"], twin.read(ak)[0]["storage_root32"])
        assert db_over(ctx, f).dump() == db_over(ctx, st).dump(back=back)
        want = state_nodes(oracle.keccak256, m)
        checked(oracle, f, m, around(m, rng, [big, doomed, reborn] + keys[3:8], diverge=False)[::5], want)
        akeys, slots = request_for(rng, m, [big, doomed, reborn] + [keys[3 + int(i)] for i in rng.choice(5997, 200, replace=False)],
                                   slot_sample=40)
        r = proofs_checked(ctx, oracle, f, m, akeys, slots, compare=range(0, len(akeys) + len(slots), 17))
        assert r["roots32"][0].tobytes() == root
        if back:
            d = diffs[nb - back]
            nodes, off = f.witness(**d.arrays())
            tn, to = twin.witness(**d.arrays())
            assert nodes.tobytes() == tn.tobytes() and np.array_equal(off, to)
            if len(off) > 1:  # (the empty state and the empty block have no node to take a transition from)
                roots, status = ctx.transition_roots(nodes, off, np.frombuffer(root, np.uint8), **d.arrays())
                assert status[0] == 1 and roots[0].tobytes() == hist[nb - back + 1][1]
            else:
                assert root == EMPTY or not d.accounts
        f.close()
    st.close()
    twin.close()


def test_snap_at_a_pivot(ctx, oracle):
    """the trie-nodes tests' 20,000-account sequence, the pivot two blocks behind the head: fork_at(pivot) heals level by
    level to exactly the pivot's node set (W proves every account from it), and its account and storage range answers pass
    G against the pivot root; the parent keeps serving only its own root"""
    rng = np.random.default_rng(73)
    rs = host.ResidentStateDB(ctx)
    rs.set_journal(8)
    st = rs.state
    m = StateModel(oracle)
    addrs = [bytes(rng.integers(0, 256, 20, dtype=np.uint8)) for _ in range(3)]
    keys = [oracle.keccak256(a) for a in addrs] + [rkey(rng) for _ in range(20000 - 3)]
    big, doomed, reborn = keys[0], keys[1], keys[2]
    fields = lambda: (int(rng.integers(0, 1 << 20)), u32be(rng.integers(0, 1 << 60)), rkey(rng))  # noqa: E731
    writes = [(k, rkey(rng), rval(rng)) for k in keys[3:1003] for _ in range(int(rng.integers(1, 30)))]
    writes += grow_account(rng, m, doomed, 5000) + grow_account(rng, m, reborn, 300) + grow_account(rng, m, big, 1000)
    apply_checked(st, m, block(rng, m, {k: fields() for k in keys}, writes))
    models = [m.copy()]
    for target in (70000, 200, 0):
        touched = {keys[i]: fields() for i in rng.choice(np.arange(3, 20000), 40, replace=False)}
        w = grow_account(rng, m, big, target)
        small = [keys[i] for i in rng.choice(np.arange(3, 1003), 40, replace=False)]
        w += [(k, sk, ZERO32) for k in small[:20] for sk in list(m.acc[k].storage)[:2]]
        w += [(k, rkey(rng), rval(rng)) for k in small[20:]]
        apply_checked(st, m, block(rng, m, touched, w))
        models.append(m.copy())
    pm = models[1]  # the pivot: `big` holds 70,000 slots there, none at the head
    pivot = pm.root()
    assert st.root() == m.root() != pivot
    assert rs.fork_at(b"\x01" * 32) is None
    assert rs.get_trie_nodes(pivot, [[b"\x00"]]) == []  # the parent serves its own root only
    fk = rs.fork_at(pivot)
    assert fk.state.root() == pivot and fk.state.info()["journal_applies"] == 0
    healed_checked(ctx, oracle, fk.state, pm)
    assert oracle.keccak256(fk.get_trie_nodes(pivot, [[b"\x00"]])[0]) == pivot
    origin, seen = bytes(32), []
    while True:
        p = fk.account_range_proof(origin, host.MAX_KEY, 2500)
        assert host.verify_account_range(ctx, pivot, origin, p["accounts"], p["proof"]) == (True, p["more"])
        assert not host.verify_account_range(ctx, m.root(), origin, p["accounts"], p["proof"])[0]
        seen += [k for k, _ in p["accounts"]]
        if not p["more"]:
            break
        origin = host._next_key(p["accounts"][-1][0])
    assert seen == sorted(pm.acc)
    for a, k in zip(addrs, keys):
        if k not in pm.acc or not pm.acc[k].storage:
            continue
        o, got = bytes(32), {}
        while True:
            p = fk.storage_range_proof(a, o, host.MAX_KEY, 997)
            whole = o == bytes(32) and not p["more"]
            assert host.verify_storage_ranges(ctx, [(pm.storage_root(k), o, p["slots"])], p["proof"], last_is_partial=not whole) == \
                [(True, p["more"])]
            got.update(p["slots"])
            if not p["more"]:
                break
            o = host._next_key(p["slots"][-1][0])
        assert got == {sk: int.from_bytes(v, "big") for sk, v in pm.acc[k].storage.items()}
    assert st.root() == m.root()
    fk.close()
    rs.close()


def test_independence(ctx, oracle):
    """a fork and its parent move apart without touching each other; the parent may be closed first; forks of forks work"""
    rng = np.random.default_rng(75)
    st = ctx.resident_state()
    st.set_journal(8)
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(3000)]
    apply_checked(st, m, block(rng, m, {k: (1, u32be(5), ZERO32) for k in keys}, [(k, rkey(rng), rval(rng)) for k in keys[:400] for _ in range(10)]))
    hist, diffs = [m.copy()], []

    def next_block():
        touched = {keys[int(j)]: (int(rng.integers(2, 99)), u32be(rng.integers(1, 1 << 40)), rkey(rng)) for j in rng.choice(3000, 80, replace=False)}
        w = [(k, list(m.acc[k].storage)[0], ZERO32) for k in keys[:400:13]] + [(k, rkey(rng), rval(rng)) for k in keys[500:530]]
        gone = keys[2500 + len(diffs)]
        touched[gone] = (0, ZERO32, ZERO32)
        return block(rng, m, touched, w, flags={gone: DELETE})

    for _ in range(4):
        diffs.append(next_block())
        apply_checked(st, m, diffs[-1])
        hist.append(m.copy())
    k = 2
    f = st.fork(k)
    fm = hist[4 - k]
    probe = keys[:300] + keys[2500:2510] + [rkey(rng)]
    akeys, slots = request_for(rng, fm, probe, slot_sample=3)
    reads_checked(f, fm, akeys, slots)
    for _ in range(3):  # the parent moves on: three blocks, one of them reverted
        diffs.append(next_block())
        apply_checked(st, m, diffs[-1])
        hist.append(m.copy())
    assert st.revert(1) == hist[-2].root()
    m = hist[-2].copy()
    assert f.root() == fm.root()
    reads_checked(f, fm, akeys, slots)
    # the fork takes the block the parent took at that root, and reaches the root the parent recorded
    parent_root, parent_info = st.root(), st.info()
    assert f.apply(**diffs[4 - k].arrays()) == hist[4 - k + 1].root()
    assert st.root() == parent_root and st.info() == parent_info
    # the parent closed first: the fork keeps working, and forks of the fork too
    st.close()
    fm = hist[4 - k + 1]
    reads_checked(f, fm, akeys, slots)
    proofs_checked(ctx, oracle, f, fm, akeys[:50], [s for s in slots if s[0] < 50])
    f.set_journal(2)
    ff = f.fork(0)
    d = diffs[4 - k + 1]
    assert f.apply(**d.arrays()) == hist[4 - k + 2].root()
    fff = f.fork(1)
    f.close()
    assert ff.root() == fff.root() == fm.root()
    reads_checked(ff, fm, akeys, slots)
    reads_checked(fff, fm, akeys, slots)
    assert ff.apply(**d.arrays()) == hist[4 - k + 2].root()
    ff.close()
    fff.close()


def held_copies(ctx, st, d, ak, paths):
    """the witness of d, the proofs of ak and the trie nodes at paths, each taken and copied whole: the bytes a held result
    must still copy after a fork"""
    nodes, off = st.witness(**d.arrays())
    pr = st.prove(ak)
    tn = st.trie_nodes(*paths)
    return (nodes.tobytes(), off.tobytes()), {f: v.tobytes() for f, v in pr.items()}, tn


def test_parent_untouched(ctx, oracle):
    """fork leaves the parent's root and info (every field) as they were, and a held witness, proof or trie-node result still
    copies afterwards, byte-equal to one taken without a fork"""
    rng = np.random.default_rng(77)
    st = ctx.resident_state()
    st.set_journal(4)
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(2000)]
    apply_checked(st, m, block(rng, m, {k: (1, u32be(5), ZERO32) for k in keys}, [(k, rkey(rng), rval(rng)) for k in keys[:200] for _ in range(5)]))
    for i in range(3):
        apply_checked(st, m, block(rng, m, {keys[int(j)]: (2 + i, u32be(7), ZERO32) for j in rng.choice(2000, 50, replace=False)},
                                   [(k, rkey(rng), rval(rng)) for k in keys[:40]]))
    d = block(rng, m, {k: (9, u32be(9), ZERO32) for k in keys[:30]}, [(k, rkey(rng), rval(rng)) for k in keys[:10]])
    ak = np.frombuffer(b"".join(keys[:20] + [rkey(rng)]), np.uint8).copy()
    paths = (np.zeros((3, 32), np.uint8), np.array([0, 1, 2], np.uint8))
    wit_want, prf_want, tn_want = held_copies(ctx, st, d, ak, paths)
    for back in (0, 2):
        # a held witness
        rc, size = st.witness_raw(gpu.ResidentState._diff(**d.arrays()))
        assert rc == 0
        root, info = st.root(), st.info()
        st.fork(back).close()
        assert st.root() == root and st.info() == info
        nodes, off = np.zeros(max(size.nodes_bytes, 1), np.uint8), np.zeros(size.n_nodes + 1, np.uint64)
        assert st.witness_copy_raw(nodes, off) == 0
        assert (nodes[:size.nodes_bytes].tobytes(), off.tobytes()) == wit_want
        # held proofs
        q = gpu.ResidentState._request(ak)
        rc, size = st.prove_raw(q)
        assert rc == 0
        info = st.info()
        f = st.fork(back)
        assert st.info() == info
        n = len(ak) // 32
        r = dict(nodes=np.zeros(max(size.nodes_bytes, 1), np.uint8), node_off=np.zeros(size.n_nodes + 1, np.uint64),
                 node_index=np.zeros(max(size.n_refs, 1), np.uint64), proof_first=np.zeros(n + 1, np.uint64),
                 roots32=np.zeros((n, 32), np.uint8), status=np.zeros(n, np.uint8), nonce=np.zeros(n, np.uint64),
                 balance32=np.zeros((n, 32), np.uint8), storage_root32=np.zeros((n, 32), np.uint8), code_hash32=np.zeros((n, 32), np.uint8),
                 slot_vals32=np.zeros((1, 32), np.uint8))
        assert st.prove_copy_raw(gpu.Proofs(*[r[fl].ctypes.data for fl, _ in gpu.Proofs._fields_])) == 0
        r["nodes"], r["node_index"], r["slot_vals32"] = r["nodes"][:size.nodes_bytes], r["node_index"][:size.n_refs], r["slot_vals32"][:0]
        assert {fl: v.tobytes() for fl, v in r.items()} == prf_want
        f.close()
        # held trie nodes
        rc, size = st.trie_nodes_raw(gpu.ResidentState._trie_node_request(*paths))
        assert rc == 0
        info = st.info()
        f = st.fork(back)
        f.close()
        assert st.info() == info
        status, toff, data = np.zeros(3, np.uint8), np.zeros(4, np.uint64), np.zeros(max(size.nodes_bytes, 1), np.uint8)
        assert st.trie_nodes_copy_raw(gpu.TrieNodes(status.ctypes.data, toff.ctypes.data, data.ctypes.data)) == 0
        assert (list(status), [data[int(toff[i]):int(toff[i + 1])].tobytes() for i in range(3)]) == (list(tn_want[0]), tn_want[1])
    st.close()


def test_refusals(ctx, oracle):
    rng = np.random.default_rng(79)
    L = gpu._lib()
    st = ctx.resident_state()
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(200)]
    apply_checked(st, m, block(rng, m, {k: (1, u32be(5), ZERO32) for k in keys}, [(k, rkey(rng), rval(rng)) for k in keys[:20]]))
    out = C.c_void_p(12345)
    assert L.phant_gpu_resident_state_fork(None, 0, C.byref(out)) == E_INVALID and not out.value  # NULL st
    assert st.fork_raw(0, None) == E_INVALID                                                       # NULL out
    root, info = st.root(), st.info()
    out = C.c_void_p(12345)
    assert st.fork_raw(1, out) == E_INVALID and not out.value  # back on a state with journal depth 0
    st.set_journal(2)
    apply_checked(st, m, block(rng, m, {keys[0]: (7, u32be(7), ZERO32)}, []))
    root, info = st.root(), st.info()
    for back in (2, 3, 1 << 31):  # back > journal_applies
        out = C.c_void_p(12345)
        assert st.fork_raw(back, out) == E_INVALID and not out.value
        assert st.root() == root and st.info() == info
    out = C.c_void_p()
    assert st.fork_raw(1, out) == 0 and out.value
    L.phant_gpu_resident_state_close(out)
    assert st.root() == root and st.info() == info
    st.close()


def test_costs_from_the_stats(ctx, oracle):
    """fork(0) is device-to-device copies only (no launch, no host transfer) and holds no more device memory than the parent
    without its journal; fork(k) launches and moves no more than revert(k) on an identical twin; closing a fork leaves the
    parent's info as it was"""
    rng = np.random.default_rng(81)
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(20000)]
    diffs = [block(rng, m, {k: (1, u32be(5), ZERO32) for k in keys}, [(k, rkey(rng), rval(rng)) for k in keys[:2000] for _ in range(10)])]
    m.apply(diffs[0])
    for i in range(6):
        diffs.append(block(rng, m, {keys[int(j)]: (2 + i, u32be(i + 3), rkey(rng)) for j in rng.choice(20000, 2000, replace=False)},
                           [(k, rkey(rng), rval(rng)) for k in keys[:300]] + [(k, list(m.acc[k].storage)[1], ZERO32) for k in keys[300:350]]))
        m.apply(diffs[-1])

    def built():
        s = ctx.resident_state()
        s.set_journal(8)
        for d in diffs:
            s.apply(**d.arrays())
        return s

    st = built()
    assert st.root() == m.root()
    info = st.info()
    ctx.reset_stats()
    f = st.fork(0)
    s0 = ctx.stats()
    assert s0["launches"] == 0 and s0["h2d_bytes"] == 0 and s0["d2h_bytes"] == 0, s0
    assert f.root() == st.root() and f.info()["device_bytes"] <= info["device_bytes"] - info["journal_bytes"], (f.info(), info)
    f.close()
    assert st.info() == info
    for k in (1, 3, 6):
        twin = built()
        ctx.reset_stats()
        f = st.fork(k)
        sf = ctx.stats()
        ctx.reset_stats()
        assert twin.revert(k) == f.root()
        sr = ctx.stats()
        for fl in ("launches", "h2d_bytes", "d2h_bytes"):
            assert sf[fl] <= sr[fl], (k, fl, sf, sr)
        assert sf["launches"] > 0
        f.close()
        twin.close()
        assert st.info() == info
    st.close()


def test_at_size(ctx, oracle):
    """100k accounts with 1M slots at depth 8, 8 blocks: fork(8) equals a twin's revert(8) in root, counts and a sampled read
    and prove"""
    rng = np.random.default_rng(107)
    m, full = build_state(oracle, rng, 100_000, [(i * 100, 1000) for i in range(1000)])
    st, twin = ctx.resident_state(), ctx.resident_state()
    for s in (st, twin):
        assert s.apply(**full.arrays()) == m.root()
        s.set_journal(8)
    pre = m.copy()
    keys = sorted(m.acc)
    for b in range(8):
        d = block_diff(rng, m, keys, b, 3000)
        root = st.apply(**d.arrays())
        assert twin.apply(**d.arrays()) == root
        m.apply(d)
        keys = sorted(m.acc)
    assert st.root() == m.root() != pre.root()
    f = st.fork(8)
    assert twin.revert(8) == f.root() == pre.root()
    fi, ti = f.info(), twin.info()
    assert (fi["n_accounts"], fi["n_slots"]) == (ti["n_accounts"], ti["n_slots"]) == counts(pre)
    rich = [k for k in sorted(pre.acc) if pre.acc[k].storage]
    sample = list(dict.fromkeys([rich[int(i)] for i in rng.choice(len(rich), 40, replace=False)] + [keys[int(i)] for i in rng.choice(len(keys), 200, replace=False)]))
    akeys, slots = request_for(rng, pre, sample, slot_sample=20)
    reads_checked(f, pre, akeys, slots)
    proofs_checked(ctx, oracle, f, pre, akeys, slots, compare=range(0, len(akeys), 11))
    assert st.root() == m.root()
    f.close()
    twin.close()
    st.close()
