"""Execution witnesses from the resident world state (phant_gpu_resident_state_witness): every node set equals the CPU
statement tests/transition_oracle.py::witness on the Python model, T (phant_gpu_transition_roots) given it returns the root
the apply then returns, and the state is left exactly as it was."""
import numpy as np
import pytest

import transition_oracle
from phant_b200 import gpu
from phant_b200 import host
from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel, change_diff, hashed_table, load_diff
from test_gpu_resident_state import block, grow_account, rkey, rval, u32be
from test_gpu_transition_roots_at_size import block_diff, build_state

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


def node_list(nodes, off):
    return [nodes[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]


def witness_checked(ctx, oracle, st, m, d, compare=True):
    """the witness of d on st (model m, before d): byte-identical on a second call, equal to the CPU statement, ordered by
    digest without duplicates, and T on it gives the root apply(d) gives"""
    nodes, off = st.witness(**d.arrays())
    again = st.witness(**d.arrays())
    assert nodes.tobytes() == again[0].tobytes() and np.array_equal(off, again[1])
    got = node_list(nodes, off)
    digests = [oracle.keccak256(n) for n in got]
    assert digests == sorted(set(digests))
    if compare:
        assert set(got) == set(transition_oracle.witness(oracle, m, d))
    pre = st.root()
    reads_checked(ctx, m, d, nodes, off, pre)
    roots, status = ctx.transition_roots(nodes, off, np.frombuffer(pre, np.uint8), **d.arrays())
    root = st.apply(**d.arrays())
    m.apply(d)
    assert root == m.root()
    assert status[0] == 1 and roots[0].tobytes() == root
    return got


def reads_checked(ctx, m, d, nodes, off, pre):
    """P (phant_gpu_read_state) over the witness, without codes, against the model before d: every listed account, and every
    listed slot of an account the witness proves slots of (present, neither deleted nor cleared, with storage); no status 3"""
    na = len(d.accounts)
    if na == 0:
        return
    akeys = np.frombuffer(b"".join(a[0] for a in d.accounts), np.uint8).copy()
    proved = [i for i, a in enumerate(d.accounts) if a[0] in m.acc and not a[1] & (DELETE | CLEAR) and m.acc[a[0]].storage]
    slots = [(ai, sk) for ai, sk, _ in d.slots if ai in set(proved)]
    ns = len(slots)
    skeys = np.frombuffer(b"".join(sk for _, sk in slots), np.uint8).copy() if ns else None
    sacc = np.array([ai for ai, _ in slots], np.uint32) if ns else None
    out = dict(account_status=np.zeros(na, np.uint8), nonce=np.zeros(na, np.uint64), balance32=np.zeros((na, 32), np.uint8),
               storage_root32=np.zeros((na, 32), np.uint8), code_hash32=np.zeros((na, 32), np.uint8), slot_status=np.zeros(max(ns, 1), np.uint8),
               slot_vals32=np.zeros((max(ns, 1), 32), np.uint8))
    data = nodes if len(nodes) else np.zeros(1, np.uint8)
    ctx.read_state(len(off) - 1, data, off, na, akeys, np.frombuffer(pre, np.uint8).copy(), 1, ns, skeys, sacc, 0, None, None, **out)
    for i, a in enumerate(d.accounts):
        acc = m.acc.get(a[0])
        if acc is None:
            assert out["account_status"][i] == 2, i
            continue
        assert out["account_status"][i] == 1, i
        assert int(out["nonce"][i]) == acc.nonce and out["balance32"][i].tobytes() == acc.balance
        assert out["storage_root32"][i].tobytes() == m.storage_root(a[0]) and out["code_hash32"][i].tobytes() == acc.code_hash
    for j, (ai, sk) in enumerate(slots):
        v = m.acc[d.accounts[ai][0]].storage.get(sk)
        assert out["slot_status"][j] == (1 if v is not None else 2), j
        assert out["slot_vals32"][j].tobytes() == (v if v is not None else ZERO32)


def test_fixtures_witness_equals_the_cpu_statement(ctx, oracle, golden):
    g = golden("fixture_states.json.gz")
    n = 0
    for t in g["tests"]:
        pre, post = hashed_table(oracle.keccak256, g["tables"][t["pre"]]), hashed_table(oracle.keccak256, g["tables"][t["post"]])
        st = ctx.resident_state()
        m = StateModel(oracle)
        st.apply(**load_diff(pre).arrays())
        m.apply(load_diff(pre))
        assert st.root().hex() == t["pre_root"]
        witness_checked(ctx, oracle, st, m, change_diff(pre, post))
        assert st.root().hex() == t["post_root"], t["name"]
        st.close()
        n += 1
    assert n == 84


def test_block_sequence(ctx, oracle):
    rng = np.random.default_rng(21)
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
    assert st.root() == m.root()
    blocks = []
    for target in (1000, 70000, 200, 0):  # `big`: L 0 -> 1 -> 3 -> 0, then no storage
        touched = {keys[i]: fields() for i in rng.choice(np.arange(3, 20000), 40, replace=False)}
        w = grow_account(rng, m, big, target)
        small = [keys[i] for i in rng.choice(np.arange(3, 1003), 40, replace=False)]
        w += [(k, sk, ZERO32) for k in small[:20] for sk in list(m.acc[k].storage)[:2]]  # deletes that collapse branches
        w += [(k, rkey(rng), rval(rng)) for k in small[20:]]
        blocks.append(block(rng, m, touched, w))
        witness_checked(ctx, oracle, st, m, blocks[-1])
    # `doomed` destroyed with 5,000 slots, `reborn` destroyed and re-created, accounts deleted next to each other
    gone = sorted(keys[3000:3400])[100:110]
    d = block(rng, m, {doomed: (0, ZERO32, ZERO32), reborn: fields(), **{k: (0, ZERO32, ZERO32) for k in gone}},
              [(reborn, rkey(rng), rval(rng)) for _ in range(40)], flags={doomed: DELETE, reborn: CLEAR, **{k: DELETE for k in gone}})
    witness_checked(ctx, oracle, st, m, d)
    witness_checked(ctx, oracle, st, m, Diff())  # an empty block
    for _ in range(6):
        touched = {keys[i]: fields() for i in rng.choice(np.arange(3, 20000), 30, replace=False)}
        live = [k for k in keys[3:1003] if k in m.acc and m.acc[k].storage]
        w = [(k, sk, ZERO32 if rng.integers(0, 2) else rval(rng)) for k in live[:50] for sk in list(m.acc[k].storage)[:2]]
        flags = {keys[int(i)]: DELETE for i in rng.choice(np.arange(5000, 20000), 5, replace=False) if keys[int(i)] in m.acc}
        for k in flags:
            touched[k] = (0, ZERO32, ZERO32)
        witness_checked(ctx, oracle, st, m, block(rng, m, touched, w, flags=flags))
    st.close()


def test_edge_cases(ctx, oracle):
    rng = np.random.default_rng(5)
    # the empty state: no node
    st = ctx.resident_state()
    m = StateModel(oracle)
    k0 = rkey(rng)
    assert witness_checked(ctx, oracle, st, m, Diff([(k0, 0, 1, u32be(1), ZERO32)], [(0, rkey(rng), u32be(3))])) == []
    st.close()
    # crafted slot keys that break the dense-top premise, then deletes of the smallest and largest keys and of a whole bucket
    st = ctx.resident_state()
    m = StateModel(oracle)
    a, b, c = rkey(rng), rkey(rng), rkey(rng)
    one = lambda: bytes([int(rng.integers(1, 0x80))]).rjust(32, b"\x00")  # noqa: E731
    ka = [bytes([0xa0 | int(rng.integers(0, 16))]) + rkey(rng)[1:] for _ in range(300)]
    kb = [b"\x5c" + rkey(rng)[1:] for _ in range(5000)]
    kc = []
    for i in range(150):
        base = b"\x77" * 28 + bytes([i]) + rkey(rng)[:2]
        kc += [base + bytes([0x10]), base + bytes([0x11])]
    others = [rkey(rng) for _ in range(400)]
    w = [(a, k, one()) for k in ka] + [(b, k, one()) for k in kb] + [(c, k, one()) for k in kc]
    d = block(rng, m, {a: (1, u32be(1), ZERO32), b: (2, u32be(2), ZERO32), c: (3, u32be(3), ZERO32), **{k: (1, u32be(1), ZERO32) for k in others}}, w)
    st.apply(**d.arrays())
    m.apply(d)
    for _ in range(2):
        w = [(a, ka[i], one()) for i in rng.choice(300, 20, replace=False)] + [(b, kb[i], ZERO32) for i in rng.choice(5000, 30, replace=False)]
        w += [(b, rkey(rng), one()) for _ in range(10)] + [(c, kc[i], ZERO32) for i in rng.choice(300, 10, replace=False)]
        w = list({(x[0], x[1]): x for x in w}.values())
        witness_checked(ctx, oracle, st, m, block(rng, m, {}, w))
    sa = sorted(m.acc[a].storage)
    witness_checked(ctx, oracle, st, m, block(rng, m, {}, [(a, sa[0], ZERO32), (a, sa[-1], ZERO32)]))  # one neighbour each
    bucket = [k for k in sorted(m.acc[b].storage) if k[1] >> 4 == 3]
    witness_checked(ctx, oracle, st, m, block(rng, m, {}, [(b, k, ZERO32) for k in bucket]))            # a whole bucket
    acc = sorted(m.acc)
    witness_checked(ctx, oracle, st, m, block(rng, m, {acc[0]: (0, ZERO32, ZERO32), acc[-1]: (0, ZERO32, ZERO32)}, [],
                                              flags={acc[0]: DELETE, acc[-1]: DELETE}))
    ghosts = [rkey(rng) for _ in range(5)]  # absent keys only
    witness_checked(ctx, oracle, st, m, block(rng, m, {g: (0, ZERO32, ZERO32) for g in ghosts[:3]} | {ghosts[3]: (1, u32be(1), ZERO32)},
                                              [(ghosts[3], rkey(rng), ZERO32)], flags={g: DELETE for g in ghosts[:3]}))
    acc = sorted(m.acc)  # every account deleted
    witness_checked(ctx, oracle, st, m, block(rng, m, {k: (0, ZERO32, ZERO32) for k in acc}, [], flags={k: DELETE for k in acc}))
    assert st.root() == transition_oracle.EMPTY_ROOT
    st.close()


def loaded(ctx, oracle, seed, n=2000):
    rng = np.random.default_rng(seed)
    st = ctx.resident_state()
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(n)]
    d = block(rng, m, {k: (1, u32be(5), ZERO32) for k in keys}, [(k, rkey(rng), rval(rng)) for k in keys[:500] for _ in range(8)])
    st.apply(**d.arrays())
    m.apply(d)
    return rng, st, m, keys


def test_state_is_unchanged_by_a_witness(ctx, oracle):
    rng, st, m, keys = loaded(ctx, oracle, 9)
    _, twin, _, _ = loaded(ctx, oracle, 9)
    st.set_journal(4)
    twin.set_journal(4)
    fixed = {k: v for k, v in st.info().items() if k != "device_bytes"}
    roots = []
    for i in range(6):
        touched = {keys[int(j)]: (2, u32be(i), ZERO32) for j in rng.choice(2000, 50, replace=False)}
        w = [(k, list(m.acc[k].storage)[0], ZERO32) for k in keys[i * 20:i * 20 + 20]]
        d = block(rng, m, touched, w)
        root = st.root()
        st.witness(**d.arrays())
        assert st.root() == root
        assert {k: v for k, v in st.info().items() if k != "device_bytes"} == fixed
        r1, s1 = st.apply(**d.arrays(), storage_roots=True)
        r2, s2 = twin.apply(**d.arrays(), storage_roots=True)
        m.apply(d)
        assert r1 == r2 == m.root() and np.array_equal(s1, s2)
        roots.append(r1)
        fixed = {k: v for k, v in st.info().items() if k != "device_bytes"}
    # revert after witness calls, then the witness equals a twin brought to the same contents by applies alone
    probe = block(rng, m, {keys[k]: (7, u32be(7), ZERO32) for k in range(0, 2000, 40)}, [(keys[3], list(m.acc[keys[3]].storage)[0], ZERO32)])
    st.witness(**probe.arrays())
    assert st.revert(2) == roots[3]
    _, fresh, _, _ = loaded(ctx, oracle, 9)
    rng3, spare, m3, _ = loaded(ctx, oracle, 9)
    spare.close()
    st2_root = None
    for i in range(4):  # replay the first four blocks on the fresh state
        touched = {keys[int(j)]: (2, u32be(i), ZERO32) for j in rng3.choice(2000, 50, replace=False)}
        w = [(k, list(m3.acc[k].storage)[0], ZERO32) for k in keys[i * 20:i * 20 + 20]]
        d = block(rng3, m3, touched, w)
        st2_root = fresh.apply(**d.arrays())
        m3.apply(d)
    assert st2_root == roots[3] == st.root()
    a, b = st.witness(**probe.arrays()), fresh.witness(**probe.arrays())
    assert a[0].tobytes() == b[0].tobytes() and np.array_equal(a[1], b[1])
    for s in (st, twin, fresh):
        s.close()


def test_refusals_hold_nothing(ctx, oracle):
    rng, st, m, keys = loaded(ctx, oracle, 4, 300)
    k1, k2, s1 = rkey(rng), rkey(rng), rkey(rng)
    f = (1, u32be(9), ZERO32)
    bad = [Diff([(k1,) + (0,) + f, (k1,) + (0,) + f]),
           Diff([(k1, 0) + f], [(0, s1, u32be(1)), (0, s1, u32be(2))]),
           Diff([(k1, 0) + f], [(1, s1, u32be(1))]),
           Diff([(k1, DELETE) + f, (k2, 0) + f], [(0, s1, u32be(1))]),
           Diff([(k1, 4) + f])]
    nodes, off = np.zeros(1 << 16, np.uint8), np.zeros(1 << 12, np.uint64)
    for d in bad:
        with pytest.raises(gpu.PhantGpuError) as e:
            st.witness(**d.arrays())
        assert e.value.code == -1
        assert st.witness_copy_raw(nodes, off) == -1
    assert st.witness_copy_raw(nodes, off) == -1  # nothing held
    good = Diff([(keys[0], 0) + f])
    for after in (lambda: st.set_journal(2), lambda: st.apply(**good.arrays()), lambda: st.revert(1)):
        rc, size = st.witness_raw(gpu.ResidentState._diff(**good.arrays()))
        assert rc == 0 and size.n_nodes > 0
        after()
        assert st.witness_copy_raw(nodes, off) == -1
    st.close()


def test_work_from_the_stats(ctx, oracle):
    rng = np.random.default_rng(12)
    st = ctx.resident_state()
    m = StateModel(oracle)
    big = rkey(rng)
    keys = [rkey(rng) for _ in range(3000)]
    w = [(big, rkey(rng), rval(rng)) for _ in range(1_000_000)]
    d = block(rng, m, {big: (1, u32be(1), ZERO32), **{k: (1, u32be(1), ZERO32) for k in keys}}, w)
    st.apply(**d.arrays())
    one = Diff([(big, 0, 1, u32be(1), ZERO32)], [(0, w[5][1], u32be(9))])
    ctx.reset_stats()
    st.witness(**one.arrays())
    s = ctx.stats()
    assert s["keccak_msgs"] < 2000 and s["h2d_bytes"] < 1024, s
    launches = []
    for n in (10, 2000):
        dd = Diff([(k, 0, 2, u32be(2), ZERO32) for k in keys[:n]])
        ctx.reset_stats()
        st.witness(**dd.arrays())
        launches.append(ctx.stats()["launches"])
    assert launches[1] < 2 * launches[0], launches
    sizes = []
    for i in range(100):
        dd = Diff([(k, 0, 2, u32be(2), ZERO32) for k in keys[(i * 20) % 2900:(i * 20) % 2900 + 20]])
        st.witness(**dd.arrays())
        sizes.append(st.info()["device_bytes"])
    assert max(sizes) <= 2 * sizes[0], sizes
    st.close()


def fixture_touched(pre_t, post_t):
    """a fixture's block as ResidentStateDB.apply takes it: touched accounts (None: destroyed) and the slots written"""
    acct = lambda a: host.AccountState(a["nonce"], int(a["balance"] or "0", 16), bytes.fromhex(a["code"]),  # noqa: E731
                                       {int(k, 16): int(v, 16) for k, v in a["storage"].items() if int(v, 16)})
    old = {bytes.fromhex(a["address"]): acct(a) for a in pre_t}
    new = {bytes.fromhex(a["address"]): acct(a) for a in post_t}
    touched, slots = {}, {}
    for addr in set(old) | set(new):
        o, n = old.get(addr), new.get(addr)
        if n is None:
            touched[addr] = None
            continue
        writes = {k: v for k, v in n.storage.items() if (o.storage.get(k) if o else None) != v}
        writes.update({k: 0 for k in (o.storage if o else {}) if k not in n.storage})
        if o and (o.nonce, o.balance, o.code) == (n.nonce, n.balance, n.code) and not writes:
            continue
        touched[addr], slots[addr] = n, writes
    return old, touched, slots


def test_fixtures_through_the_host_layer(ctx, oracle, golden):
    """host.ResidentStateDB.witness on every fixture: the CPU statement's set, and host.transition_root on the blob it makes
    gives the header's post root"""
    g = golden("fixture_states.json.gz")
    for t in g["tests"]:
        pre_t, post_t = g["tables"][t["pre"]], g["tables"][t["post"]]
        old, touched, slots = fixture_touched(pre_t, post_t)
        rs = host.ResidentStateDB(ctx)
        if old:
            assert rs.apply(old).hex() == t["pre_root"], t["name"]
        m = StateModel(oracle)
        pre, post = hashed_table(oracle.keccak256, pre_t), hashed_table(oracle.keccak256, post_t)
        m.apply(load_diff(pre))
        nodes = rs.witness(touched, slots)
        assert set(nodes) == set(transition_oracle.witness(oracle, m, change_diff(pre, post))), t["name"]
        if touched:
            codes = [s.code for s in touched.values() if s is not None and s.code]
            root, status = host.transition_root(ctx, bytes.fromhex(t["pre_root"]), host.encode_witness([], codes, nodes), touched, slots)
            assert status == 1 and root.hex() == t["post_root"], t["name"]
        assert rs.apply(touched, slots).hex() == t["post_root"], t["name"]
        rs.close()


def test_100k_accounts_1m_slots_64_blocks(ctx, oracle):
    """at size: every block's witness, through T, gives the root its apply gives; four of them equal the CPU statement"""
    rng = np.random.default_rng(101)
    m, full = build_state(oracle, rng, 100_000, [(i * 100, 1000) for i in range(1000)])
    st = ctx.resident_state()
    assert st.apply(**full.arrays()) == m.root()
    keys = sorted(m.acc)
    for b in range(64):
        d = block_diff(rng, m, keys, b, 3000)
        nodes, off = st.witness(**d.arrays())
        if b % 16 == 5:
            assert set(node_list(nodes, off)) == set(transition_oracle.witness(oracle, m, d)), b
        pre = st.root()
        roots, status = ctx.transition_roots(nodes, off, np.frombuffer(pre, np.uint8), **d.arrays())
        root = st.apply(**d.arrays())
        m.apply(d)
        assert status[0] == 1 and roots[0].tobytes() == root, b
        keys = sorted(m.acc)
    assert st.root() == m.root()
    st.close()
