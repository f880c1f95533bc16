"""Snap range answers from the resident world state (phant_gpu_resident_state_snap_ranges: GetAccountRange and
GetStorageRanges with byte budgets, slim account bodies and boundary proofs): every answer equals the CPU statement
(tests/snap_serve_model.py) byte for byte -- entries, bodies, served accounts and proof lists in wire order -- and G
(phant_gpu_verify_ranges, through host.verify_snap_account_range / verify_snap_storage_ranges) accepts it, with `more` set
exactly when the answer stopped before the trie's end.  A whole state synced through the host layer rebuilds the same root;
batches equal their requests answered alone; the state is left as it was, and the one-result rules hold."""
import numpy as np
import pytest

from phant_b200 import gpu
from phant_b200 import host
from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel, hashed_table, load_diff
from snap_serve_model import FF, ZERO, Prover, account_answer, storage_answer
from test_gpu_resident_state import block, grow_account, rkey, rval, u32be
from test_gpu_transition_roots_at_size import build_state

pytestmark = pytest.mark.gpu

BUDGETS = (0, 1, 36, 37, 100, 500, 4096, 2 << 20, 1 << 63)


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


def add(k, d):
    return ((int.from_bytes(k, "big") + d) % (1 << 256)).to_bytes(32, "big")


def loaded(ctx, oracle, diff):
    st, m = ctx.resident_state(), StateModel(oracle)
    st.apply(**diff.arrays())
    m.apply(diff)
    return st, m


def compare(oracle, st, m, ar, sr, verify=True):
    """one device call with account requests ar [(origin, limit, bytes)] and storage requests sr [([accounts], origin, limit,
    bytes)]: equal to the model, accepted by G; the state is unchanged"""
    root, info = st.root(), st.info()
    got = st.snap_ranges(ar, sr)
    assert st.root() == root
    assert {k: v for k, v in st.info().items() if k != "device_bytes"} == {k: v for k, v in info.items() if k != "device_bytes"}
    pv = Prover(oracle, m)
    keys = sorted(m.acc)
    for i, (o, lim, b) in enumerate(ar):
        want = account_answer(m, pv, o, lim, b)
        assert (got["accounts"][i], got["proofs"][i]) == want, (i, o.hex(), lim.hex(), b)
        if verify:
            ok, more = host.verify_snap_account_range(st.ctx, root, o, *want)
            assert ok, (i, o.hex(), b)
            assert more == bool(want[0] and want[0][-1][0] < keys[-1]), (i, o.hex(), b)
    for j, (accts, o, lim, b) in enumerate(sr):
        want = storage_answer(m, pv, accts, o, lim, b)
        assert (got["slots"][j], got["proofs"][len(ar) + j]) == want, (j, o.hex(), lim.hex(), b)
        if verify and want[0] and (o != ZERO or lim == FF):  # a zero origin with a limit is cut by the limit, with no proof
            roots = [m.storage_root(a) if a in m.acc else host.EMPTY_MPT_ROOT for a in accts[:len(want[0])]]
            res = host.verify_snap_storage_ranges(st.ctx, roots, o, *want)
            assert all(ok for ok, _ in res), (j, res)
            for i, (lst, (_, more)) in enumerate(zip(want[0], res)):
                a = m.acc.get(accts[i])
                last = max(a.storage) if a and a.storage else None
                if want[1] and i + 1 == len(want[0]):
                    assert more == bool(lst and last is not None and lst[-1][0] < last), (j, i)
                else:
                    assert not more
    return got


def requests_over(m, rng, n_acc=24, n_sto=16):
    """account requests at every key's neighbours (a sample) and storage requests over accounts with storage"""
    keys = sorted(m.acc)
    rich = [k for k in keys if m.acc[k].storage]
    ar = [(ZERO, FF, b) for b in BUDGETS]
    for k in (keys if len(keys) <= n_acc else [keys[i] for i in rng.choice(len(keys), n_acc, replace=False)]):
        for o in (add(k, -1), k, add(k, 1)):
            ar.append((o, FF, int(rng.choice(BUDGETS))))
        ar.append((k, k, 1 << 20))
        ar.append((k, add(k, -1), 1 << 20))  # origin above limit
    if keys:
        ar.append((add(keys[-1], 1), FF, 1000))  # origin above every key
    sr = []
    for _ in range(n_sto):
        accts = [rich[i] for i in rng.integers(0, len(rich), int(rng.integers(1, 5)))] if rich else []
        accts.insert(int(rng.integers(0, len(accts) + 1)), rkey(rng))  # an absent account in the middle
        if len(keys) > len(rich):
            accts.insert(int(rng.integers(0, len(accts) + 1)), [k for k in keys if not m.acc[k].storage][0])  # no storage
        first = m.acc.get(accts[0])
        sk = sorted(first.storage) if first else []
        o = sk[int(rng.integers(0, len(sk)))] if sk and rng.random() < 0.5 else ZERO
        lim = sk[int(rng.integers(0, len(sk)))] if sk and rng.random() < 0.3 else FF
        sr.append((accts, o, lim, int(rng.choice(BUDGETS))))
    return ar, sr


def test_fixtures(ctx, oracle, golden):
    g = golden("fixture_states.json.gz")
    rng = np.random.default_rng(71)
    n = 0
    for name in sorted(g["tables"]):
        st, m = loaded(ctx, oracle, load_diff(hashed_table(oracle.keccak256, g["tables"][name])))
        ar, sr = requests_over(m, rng)
        compare(oracle, st, m, ar, sr)
        st.close()
        n += 1
    assert n >= 84


def test_larger_state_and_crafted_keys(ctx, oracle):
    """2,000 accounts, accounts with 1..3,000 slots, keys sharing long prefixes (extensions, embedded-leaf depths)"""
    rng = np.random.default_rng(72)
    _, d0 = build_state(oracle, rng, 2000, [(0, 3000), (1, 400), (2, 40), (3, 1), (4, 2)])
    diff = d0
    shared = b"\x42" * 31
    diff.accounts += [(shared + bytes([i]), 0, i, (0).to_bytes(32, "big"), host.EMPTY_CODE_HASH) for i in (1, 2, 0x10, 0x11)]
    diff.accounts.append((shared + b"\x12", 0, (1 << 64) - 1, b"\xff" * 32, host.EMPTY_CODE_HASH))  # the widest slim body
    k0 = diff.accounts[0][0]
    diff.slots += [(0, b"\x77" * 31 + bytes([i]), (5).to_bytes(32, "big")) for i in (0x10, 0x11, 0x20)]  # embedded leaves
    st, m = loaded(ctx, oracle, diff)
    assert k0 in m.acc
    ar, sr = requests_over(m, rng, 40, 40)
    rich = sorted((k for k in m.acc if m.acc[k].storage), key=lambda k: -len(m.acc[k].storage))
    for b in (0, 1, 33, 4096, 65536, 512 << 10, 2 << 20):
        sr.append((rich[:6], ZERO, FF, b))
        sk = sorted(m.acc[rich[0]].storage)
        sr.append((rich[:3], sk[100], FF, b))
        sr.append((rich[1:4] + rich[:1], ZERO, FF, b))  # the big account cut after smaller ones
    compare(oracle, st, m, ar, sr)
    st.close()


def test_block_sequence(ctx, oracle):
    """the trie-nodes tests' 20,000-account block sequence: an account that grows to 70,000 slots and shrinks again, one that
    is destroyed, one re-created, accounts deleted; answered after the load and after every block"""
    rng = np.random.default_rng(77)
    st = ctx.resident_state()
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(20000)]
    big, doomed, reborn = keys[0], keys[1], keys[2]
    fields = lambda: (int(rng.integers(0, 1 << 20)), u32be(rng.integers(0, 1 << 60)), rkey(rng))  # noqa: E731
    writes = [(k, rkey(rng), rval(rng)) for k in keys[3:1003] for _ in range(int(rng.integers(1, 30)))]
    writes += grow_account(rng, m, doomed, 5000) + grow_account(rng, m, reborn, 300)
    blocks = [block(rng, m, {k: fields() for k in keys}, writes)]

    def step(d):
        st.apply(**d.arrays())
        m.apply(d)
        ar, sr = requests_over(m, rng, 12, 12)
        for b in (4096, 512 << 10):
            sr.append(([big, doomed, reborn] + keys[3:8], ZERO, FF, b))
        compare(oracle, st, m, ar, sr)
    step(blocks[0])
    for target in (70000, 200):
        touched = {keys[i]: fields() for i in rng.choice(np.arange(3, 20000), 40, replace=False)}
        w = grow_account(rng, m, big, target)
        small = [keys[i] for i in rng.choice(np.arange(3, 1003), 40, replace=False)]
        w += [(k, sk, ZERO32) for k in small[:20] for sk in list(m.acc[k].storage)[:2]]
        w += [(k, rkey(rng), rval(rng)) for k in small[20:]]
        step(block(rng, m, touched, w))
    gone = sorted(keys[3000:3400])[100:110]
    step(block(rng, m, {doomed: (0, ZERO32, ZERO32), reborn: fields(), **{k: (0, ZERO32, ZERO32) for k in gone}},
               [(reborn, rkey(rng), rval(rng)) for _ in range(40)], flags={doomed: DELETE, reborn: CLEAR, **{k: DELETE for k in gone}}))
    st.close()


def test_empty_state(ctx, oracle):
    st, m = loaded(ctx, oracle, Diff())
    compare(oracle, st, m, [(ZERO, FF, 0), (ZERO, FF, 1000), (FF, ZERO, 5)], [([rkey(np.random.default_rng(1))], ZERO, FF, 100),
                                                                             ([rkey(np.random.default_rng(2))], FF, FF, 100)])
    got = st.snap_ranges()
    assert got["accounts"] == [] and got["slots"] == [] and got["proofs"] == []
    st.close()


def test_batch_equals_alone_and_launches(ctx, oracle):
    rng = np.random.default_rng(73)
    _, d0 = build_state(oracle, rng, 3000, [(i, 50) for i in range(40)])
    st, m = loaded(ctx, oracle, d0)
    keys = sorted(m.acc)
    rich = [k for k in keys if m.acc[k].storage]
    ar = [(keys[int(i)], FF, int(rng.choice((100, 4096, 20000)))) for i in rng.integers(0, len(keys), 600)]
    sr = [([rich[int(i)] for i in rng.integers(0, len(rich), 4)], ZERO, FF, int(rng.choice((100, 1000, 4096)))) for _ in range(400)]
    ctx.reset_stats()
    big = st.snap_ranges(ar, sr)
    launches_big = ctx.stats()["launches"]
    ctx.reset_stats()
    st.snap_ranges(ar[:6], sr[:4])
    launches_small = ctx.stats()["launches"]
    assert launches_big < 2 * launches_small, (launches_big, launches_small)
    for i in list(range(0, 600, 37)):
        one = st.snap_ranges([ar[i]])
        assert one["accounts"][0] == big["accounts"][i] and one["proofs"][0] == big["proofs"][i]
    for j in list(range(0, 400, 29)):
        one = st.snap_ranges([], [sr[j]])
        assert one["slots"][0] == big["slots"][j] and one["proofs"][0] == big["proofs"][600 + j]
    compare(oracle, st, m, ar[::20], sr[::20], verify=False)
    st.close()


def test_sync_from_snap(ctx, oracle):
    """a whole state walked through snap_account_range and snap_storage_ranges (64 accounts per request, cut accounts
    continued), every answer checked with G, then loaded into a fresh state with one apply: the same root"""
    rng = np.random.default_rng(74)
    _, d0 = build_state(oracle, rng, 1500, [(i, int(rng.integers(1, 600))) for i in range(0, 300, 3)])
    db = host.ResidentStateDB(ctx)
    db.state.apply(**d0.arrays())
    root = db.state.root()
    accounts, origin = [], ZERO
    while True:
        got, proof = db.snap_account_range(root, origin, FF, 16 << 10)
        ok, more = host.verify_snap_account_range(ctx, root, origin, got, proof)
        assert ok and got
        accounts += got
        if not more:
            break
        origin = add(got[-1][0], 1)
    full = {k: host.decode_slim_account(b) for k, b in accounts}
    assert sorted(full) == sorted(a[0] for a in d0.accounts)
    storage = {k: {} for k in full}
    pending = [k for k, v in full.items() if v[2] != host.EMPTY_MPT_ROOT]
    o = ZERO
    while pending:
        batch = pending[:64]
        lists, proof = db.snap_storage_ranges(root, batch, o, FF, 32 << 10)
        res = host.verify_snap_storage_ranges(ctx, [full[a][2] for a in batch[:len(lists)]], o, lists, proof)
        assert lists and all(ok for ok, _ in res)
        for a, lst in zip(batch, lists):
            storage[a].update((k, (v if v[0] < 0x80 else v[1:]).rjust(32, b"\x00")) for k, v in lst)
        done = len(lists)
        if proof and res[-1][1]:  # the last account was cut: continue it
            o = add(lists[-1][-1][0], 1) if lists[-1] else o
            done -= 1
        else:
            o = ZERO
        pending = pending[done:]
    fresh = ctx.resident_state()
    d = Diff([(k, 0, v[0], v[1].to_bytes(32, "big"), v[3]) for k, v in full.items()])
    for i, (k, _, _, _, _) in enumerate(d.accounts):
        d.slots += [(i, sk, sv) for sk, sv in storage[k].items()]
    assert fresh.apply(**d.arrays()) == root
    fresh.close()
    db.close()


def test_at_a_pivot(ctx, oracle):
    """a fork at back 4 serves the answers of that root"""
    rng = np.random.default_rng(75)
    st, m = ctx.resident_state(), StateModel(oracle)
    st.set_journal(8)
    hist = []
    keys = [rkey(rng) for _ in range(200)]
    for b in range(6):
        d = Diff([(k, 0, b * 1000 + i, (b + 1).to_bytes(32, "big"), rkey(rng)) for i, k in enumerate(keys[b * 30:b * 30 + 60])],
                 [(i, rkey(rng), rval(rng)) for i in range(0, len(keys[b * 30:b * 30 + 60]), 7)])
        st.apply(**d.arrays())
        m.apply(d)
        hist.append(m.copy())
    f = st.fork(4)
    pm = hist[1]
    assert f.root() == pm.root()
    rich = [k for k in pm.acc if pm.acc[k].storage]
    compare(oracle, f, pm, [(ZERO, FF, 1000), (sorted(pm.acc)[5], FF, 300)], [(rich[:3], ZERO, FF, 40)])
    f.close()
    st.close()


def raw_request(**over):
    q = gpu.ResidentState._snap_request([(ZERO, FF, 100)], [([b"\x01" * 32], ZERO, FF, 100)])
    for k, v in over.items():
        setattr(q, k, v)
    return q


def test_refusals_and_one_result(ctx, oracle):
    rng = np.random.default_rng(76)
    _, d0 = build_state(oracle, rng, 300, [(0, 30)])
    st, m = loaded(ctx, oracle, d0)
    root = st.root()
    bad_first = np.array([1, 1], np.uint64)
    dec_first = np.array([0, 2, 1], np.uint64)
    for over in (dict(account_origin32=None), dict(account_bytes=None), dict(storage_first=None), dict(storage_accounts32=None),
                 dict(storage_first=bad_first.ctypes.data), dict(n_account_requests=(1 << 28) + 1), dict(n_storage_requests=(1 << 28) + 1)):
        q = raw_request(**over)
        q._k2 = (bad_first, dec_first)
        rc, _ = st.snap_ranges_raw(q)
        assert rc == -1, over  # PHANT_GPU_E_INVALID
        assert st.snap_ranges_copy_raw(gpu.SnapRanges()) == -1
    q = raw_request(n_storage_requests=2, storage_first=dec_first.ctypes.data)
    assert st.snap_ranges_raw(q)[0] == -1
    # one result at a time
    key = np.frombuffer(sorted(m.acc)[0], np.uint8)
    want = st.snap_ranges([(ZERO, FF, 100)], [([b"\x01" * 32], ZERO, FF, 100)])
    assert st.snap_ranges_raw(raw_request())[0] == 0
    st.prove(key)
    assert st.snap_ranges_copy_raw(gpu.SnapRanges()) == -1
    rc, size = st.snap_ranges_raw(raw_request())
    assert rc == 0
    assert st.prove_copy_raw(gpu.Proofs()) == -1
    assert st.trie_nodes_copy_raw(gpu.TrieNodes()) == -1
    assert st.witness_copy_raw(None, None) == -1
    st.read(key)
    st.range([(ZERO, FF, 3)])
    st.codes(np.zeros(32, np.uint8))
    st.fork(0).close()
    # the held result still copies after read, range, codes and a fork
    z = lambda k, t=np.uint64: np.zeros(max(int(k), 1), t)  # noqa: E731
    r = dict(account_first=z(2), account_keys32=z(32 * size.n_accounts, np.uint8), account_body_off=z(size.n_accounts + 1),
             account_bodies=z(size.account_bytes, np.uint8), served_first=z(2), slot_first=z(size.n_served + 1),
             slot_keys32=z(32 * size.n_slots, np.uint8), slot_body_off=z(size.n_slots + 1), slot_bodies=z(size.slot_bytes, np.uint8),
             proof_first=z(3), node_index=z(size.n_refs), nodes=z(size.nodes_bytes, np.uint8), node_off=z(size.n_nodes + 1))
    assert st.snap_ranges_copy_raw(gpu.SnapRanges(*[gpu._ptr(r[f]) for f, _ in gpu.SnapRanges._fields_])) == 0
    assert st.snap_ranges_copy_raw(gpu.SnapRanges()) == -1  # copied: nothing held
    n_acc = int(r["account_first"][1])
    assert n_acc == len(want["accounts"][0]) and int(r["served_first"][1]) == len(want["slots"][0])
    assert [r["account_keys32"][32 * e:32 * e + 32].tobytes() for e in range(n_acc)] == [k for k, _ in want["accounts"][0]]
    assert st.snap_ranges_raw(raw_request())[0] == 0
    st.trie_nodes(np.zeros(32, np.uint8), np.zeros(1, np.uint8))
    assert st.snap_ranges_copy_raw(gpu.SnapRanges()) == -1
    assert st.snap_ranges_raw(raw_request())[0] == 0
    st.apply(**Diff().arrays())
    assert st.snap_ranges_copy_raw(gpu.SnapRanges()) == -1
    # witness and set_journal drop it; snap_ranges drops a held witness or trie-node result
    wd = gpu.ResidentState._diff(**Diff([(sorted(m.acc)[0], 0, 1, bytes(32), bytes(32))]).arrays())
    assert st.snap_ranges_raw(raw_request())[0] == 0
    assert st.witness_raw(wd)[0] == 0
    assert st.snap_ranges_copy_raw(gpu.SnapRanges()) == -1
    assert st.snap_ranges_raw(raw_request())[0] == 0
    assert st.witness_copy_raw(None, None) == -1
    tq = gpu.ResidentState._trie_node_request(np.zeros(32, np.uint8), np.zeros(1, np.uint8))
    assert st.trie_nodes_raw(tq)[0] == 0
    assert st.snap_ranges_raw(raw_request())[0] == 0
    assert st.trie_nodes_copy_raw(gpu.TrieNodes()) == -1
    st.set_journal(2)
    assert st.snap_ranges_copy_raw(gpu.SnapRanges()) == -1
    st.apply(**Diff().arrays())
    assert st.snap_ranges_raw(raw_request())[0] == 0
    st.revert(1)
    assert st.snap_ranges_copy_raw(gpu.SnapRanges()) == -1
    # host pointers only
    ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
    try:
        assert st.snap_ranges_raw(raw_request())[0] == -1
    finally:
        ctx.set_flags(0)
    assert st.snap_ranges_copy_raw(gpu.SnapRanges()) == -1
    assert st.root() == root
    st.close()
