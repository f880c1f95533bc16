"""Account and storage ranges from the resident world state (phant_gpu_resident_state_range) on the GPU, at the current root
and at every root the undo journal reaches: every range equals the Python model's slice of that block (storage roots and
`more` included), a dump loads back into the same root, range plus prove gives snap's boundary proofs, and a call changes
nothing -- not the root, the counts, the journal, nor a witness or proof result the state holds."""
import numpy as np
import pytest
import torch

from phant_b200 import gpu
from phant_b200 import host
from resident_range_model import MAX_KEY, ZERO_KEY, add, expect, ranges_over
from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel, change_diff, hashed_table, load_diff
from test_gpu_resident_state import apply_checked, block, grow_account, rkey, rval, u32be
from test_gpu_resident_state_proofs import Tries, verify
from test_gpu_transition_roots_at_size import build_state

pytestmark = pytest.mark.gpu

E_INVALID = -1
EMPTY = host.EMPTY_MPT_ROOT
ALL = (1 << 32) - 1


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


def slots_of(m, k):
    a = m.acc.get(k)
    return {sk: v for sk, v in a.storage.items() if v != ZERO32} if a else {}


def ranges_checked(st, m, aranges, sranges, back=0, root=None):
    """one range call at `back`: every range must be model m's slice, and the root `root` (default: m's)"""
    r, got = st.range(aranges, sranges, back=back)
    assert got == (root if root is not None else m.root()), back
    keys = sorted(m.acc)
    for i, (o, lim, mx) in enumerate(aranges):
        want, more = expect(keys, o, lim, mx)
        a, b = int(r["account_first"][i]), int(r["account_first"][i + 1])
        assert [r["account_keys32"][e].tobytes() for e in range(a, b)] == want, (back, i)
        assert bool(r["account_more"][i]) == more, (back, i)
        for e, k in zip(range(a, b), want):
            x = m.acc[k]
            assert (int(r["nonce"][e]), r["balance32"][e].tobytes(), r["storage_root32"][e].tobytes(), r["code_hash32"][e].tobytes()) == \
                (x.nonce, x.balance, m.storage_root(k), x.code_hash), (back, k.hex())
    for j, (ak, o, lim, mx) in enumerate(sranges):
        st_ = slots_of(m, ak)
        want, more = expect(sorted(st_), o, lim, mx)
        a, b = int(r["slot_first"][j]), int(r["slot_first"][j + 1])
        assert [r["slot_keys32"][e].tobytes() for e in range(a, b)] == want, (back, j)
        assert [r["slot_vals32"][e].tobytes() for e in range(a, b)] == [st_[k] for k in want], (back, j)
        assert bool(r["slot_more"][j]) == more, (back, j)
    return r


def whole(m, extra=()):
    """the whole account range and every account's whole storage range (plus `extra` accounts), with room for one more"""
    ks = sorted(set(m.acc) | set(extra))
    most = max([len(slots_of(m, k)) for k in ks] + [0])
    return [(ZERO_KEY, MAX_KEY, len(m.acc) + 1)], [(k, ZERO_KEY, MAX_KEY, most + 1) for k in ks]


def sub_ranges(m, rng, n):
    keys = sorted(m.acc)
    ar = ranges_over(keys, rng, n, maxes=(0, 1, 2, 5, 1 << 20))
    sr = []
    for k in keys[:20]:
        sr += [(k,) + x for x in ranges_over(sorted(slots_of(m, k)), rng, 4, maxes=(0, 1, 3, 1 << 16))]
    return ar, sr


def test_fixtures(ctx, oracle, golden):
    g = golden("fixture_states.json.gz")
    rng = np.random.default_rng(51)
    n = 0
    for t in g["tests"]:
        pre, post = hashed_table(oracle.keccak256, g["tables"][t["pre"]]), hashed_table(oracle.keccak256, g["tables"][t["post"]])
        st = ctx.resident_state()
        st.set_journal(1)
        m = StateModel(oracle)
        assert apply_checked(st, m, load_diff(pre)).hex() == t["pre_root"], t["name"]
        before = m.copy()
        apply_checked(st, m, change_diff(pre, post))
        assert m.root().hex() == t["post_root"]
        for back, h in ((0, m), (1, before)):
            ranges_checked(st, h, *whole(h, extra=set(m.acc) | set(before.acc)), back=back)
            ranges_checked(st, h, *sub_ranges(h, rng, 20), back=back)
        st.close()
        n += 1
    assert n == 84


def test_chunked_iteration(ctx, oracle):
    """origin = last + 1 with a small max walks the whole range, at back 0 and 1"""
    rng = np.random.default_rng(7)
    st = ctx.resident_state()
    st.set_journal(2)
    m = StateModel(oracle)
    ks = [rkey(rng) for _ in range(300)]
    apply_checked(st, m, Diff([(k, 0, 1, u32be(2), ZERO32) for k in ks], [(0, rkey(rng), rval(rng)) for _ in range(500)]))
    before = m.copy()
    apply_checked(st, m, block(rng, m, {rkey(rng): (1, u32be(3), ZERO32) for _ in range(100)}, [(ks[0], rkey(rng), rval(rng)) for _ in range(50)]))
    for back, h in ((0, m), (1, before)):
        for mx in (1, 7, 64):
            got, o = [], ZERO_KEY
            while True:
                r, _ = st.range([(o, MAX_KEY, mx)], back=back)
                keys = [k.tobytes() for k in r["account_keys32"]]
                got += keys
                if not r["account_more"][0]:
                    break
                o = add(keys[-1], 1)
            assert got == sorted(h.acc)
            got, o = [], ZERO_KEY
            while True:
                r, _ = st.range(storage_ranges=[(ks[0], o, MAX_KEY, mx)], back=back)
                keys = [k.tobytes() for k in r["slot_keys32"]]
                got += keys
                if not r["slot_more"][0]:
                    break
                o = add(keys[-1], 1)
            assert got == sorted(slots_of(h, ks[0]))
    st.close()


def test_block_sequence_at_every_back(ctx, oracle):
    """the revert test's blocks at depth 16, ranges at every back after every block; then revert(3), another branch, and a
    shorter journal"""
    rng = np.random.default_rng(12)
    st = ctx.resident_state()
    st.set_journal(16)
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(6000)]
    big, doomed, reborn = keys[0], keys[1], keys[2]
    fields = lambda: (int(rng.integers(0, 1 << 20)), u32be(rng.integers(0, 1 << 60)), rkey(rng))  # noqa: E731
    hist = [(m.copy(), EMPTY)]

    def step(d):
        root = apply_checked(st, m, d)
        hist.append((m.copy(), root))

    def check_all():
        n = st.info()["journal_applies"]
        for back in range(n + 1):
            h, root = hist[len(hist) - 1 - back]
            ar = [(ZERO_KEY, MAX_KEY, 1 << 16), (ZERO_KEY, MAX_KEY, 100), (keys[5], add(keys[5], 1 << 250), 40)]
            sr = [(k, ZERO_KEY, MAX_KEY, 1 << 17) for k in (big, doomed, reborn)] + [(big, keys[9], MAX_KEY, 25), (doomed, ZERO_KEY, MAX_KEY, 0)]
            ranges_checked(st, h, ar, sr, back=back, root=root)

    writes = [(k, rkey(rng), rval(rng)) for k in keys[3:1003] for _ in range(int(rng.integers(1, 10)))]
    writes += grow_account(rng, m, big, 200) + grow_account(rng, m, doomed, 5000) + grow_account(rng, m, reborn, 300)
    step(block(rng, m, {k: fields() for k in keys}, writes))
    check_all()
    for target in (1000, 5000, 70000, 5000, 1000, 200):
        touched = {keys[i]: fields() for i in rng.choice(np.arange(3, 6000), 30, replace=False)}
        w = grow_account(rng, m, big, target)
        small = [keys[i] for i in rng.choice(np.arange(3, 203), 30, replace=False)]
        w += [(k, list(m.acc[k].storage)[0], rval(rng)) for k in small if m.acc[k].storage]
        w += [(k, rkey(rng), ZERO32) for k in small[:5]]
        step(block(rng, m, touched, w))
        check_all()
    step(block(rng, m, {doomed: (0, ZERO32, ZERO32), reborn: fields()}, [(reborn, rkey(rng), rval(rng)) for _ in range(40)],
               flags={doomed: DELETE, reborn: CLEAR}))
    check_all()
    step(block(rng, m, {}, []))
    check_all()
    assert st.info()["journal_applies"] == len(hist) - 1 == 9
    assert st.revert(3) == hist[-4][1]
    del hist[-3:]
    m = hist[-1][0].copy()
    check_all()
    step(block(rng, m, {doomed: fields(), reborn: fields()}, [(doomed, rkey(rng), rval(rng)) for _ in range(50)], flags={doomed: CLEAR}))
    step(block(rng, m, {reborn: (0, ZERO32, ZERO32)}, [], flags={reborn: DELETE}))
    check_all()
    st.set_journal(2)
    check_all()
    with pytest.raises(gpu.PhantGpuError) as e:
        st.range([(ZERO_KEY, MAX_KEY, 1)], back=3)
    assert e.value.code == E_INVALID
    st.close()


def journaled(ctx, oracle, rng, n_blocks=6):
    st = ctx.resident_state()
    st.set_journal(n_blocks)
    m = StateModel(oracle)
    ks = [rkey(rng) for _ in range(400)]
    apply_checked(st, m, Diff([(k, 0, 1, u32be(2), ZERO32) for k in ks], [(i % 40, rkey(rng), rval(rng)) for i in range(2000)]))
    hist = [m.copy()]
    for _ in range(n_blocks):
        touched = {ks[int(i)]: (5, u32be(int(rng.integers(1, 1 << 40))), rkey(rng)) for i in rng.choice(400, 30, replace=False)}
        touched.update({rkey(rng): (1, u32be(1), ZERO32) for _ in range(10)})
        w = [(ks[int(i)], rkey(rng), rval(rng)) for i in rng.choice(40, 20)]
        w += [(k, list(m.acc[k].storage)[0], ZERO32) for k in ks[:3] if m.acc[k].storage]
        apply_checked(st, m, block(rng, m, touched, w, flags={ks[5]: CLEAR} if ks[5] in touched else None))
        hist.append(m.copy())
    return st, m, hist, ks


def test_round_trip(ctx, oracle):
    """dump at back 0 and back 4, loaded into a fresh state with one apply, gives exactly that root and every storage root"""
    rng = np.random.default_rng(8)
    st, m, hist, _ = journaled(ctx, oracle, rng)
    rs = host.ResidentStateDB(ctx)
    rs.state.close()
    rs.state = st
    for back in (0, 4):
        h = hist[len(hist) - 1 - back]
        table = rs.dump(back=back, chunk=97)
        _, root = st.range(back=back)
        assert table == {k: (a.nonce, a.balance, a.code_hash, slots_of(h, k)) for k, a in h.acc.items()}
        fresh = ctx.resident_state()
        d = load_diff(table)
        got, sroots = fresh.apply(**d.arrays(), storage_roots=True)
        assert got == root == h.root()
        assert [sroots[i].tobytes() for i in range(len(d.accounts))] == [h.storage_root(k) for k, *_ in d.accounts]
        fresh.close()
    rs.close()


def test_snap_composition(ctx, oracle):
    """range plus prove on {origin, last}: V accepts every boundary chain, the chains are the CPU trie's, the origin is
    present exactly when it is the first entry, and the last chain ends at the last entry's leaf"""
    rng = np.random.default_rng(9)
    st, m, _, ks = journaled(ctx, oracle, rng, n_blocks=1)
    rs = host.ResidentStateDB(ctx)
    rs.state.close()
    rs.state = st
    t = Tries(oracle, m)
    keys = sorted(m.acc)
    for o, mx in [(ZERO_KEY, 10), (keys[7], 5), (add(keys[7], 1), 5), (keys[-1], 3), (add(keys[-1], 1), 3), (keys[3], 1)]:
        p = rs.account_range_proof(o, MAX_KEY, mx)
        acc = p["accounts"]
        assert [k for k, _ in acc] == expect(keys, o, MAX_KEY, mx)[0] and p["more"] == expect(keys, o, MAX_KEY, mx)[1]
        assert p["keys"] == list(dict.fromkeys([o] + [k for k, _ in acc[-1:]]))
        pr = p["proof"]
        status, vals = verify(ctx, pr, p["keys"])
        assert (status == pr["status"]).all()
        off, data, idx, first = pr["node_off"], pr["nodes"], pr["node_index"], pr["proof_first"]
        for i, k in enumerate(p["keys"]):
            chain = [data[int(off[x]):int(off[x + 1])].tobytes() for x in idx[int(first[i]):int(first[i + 1])]]
            assert chain == t.account(k)
        assert (status[0] == 1) == (bool(acc) and acc[0][0] == o)
        if acc:
            assert vals[len(p["keys"]) - 1] == m.leaf(acc[-1][0])
    st.close()


def test_edge_cases(ctx, oracle):
    """the empty state; a state emptied by deletes with a non-empty journal"""
    rng = np.random.default_rng(10)
    st = ctx.resident_state()
    m = StateModel(oracle)
    ranges_checked(st, m, [(ZERO_KEY, MAX_KEY, 5), (MAX_KEY, ZERO_KEY, 5)], [(rkey(rng), ZERO_KEY, MAX_KEY, 5)], root=EMPTY)
    r, root = st.range()
    assert root == EMPTY and list(r["account_first"]) == [0] and list(r["slot_first"]) == [0]
    st.set_journal(3)
    ks = [rkey(rng) for _ in range(20)]
    apply_checked(st, m, Diff([(k, 0, 1, u32be(2), ZERO32) for k in ks], [(i, rkey(rng), rval(rng)) for i in range(20)]))
    full = m.copy()
    apply_checked(st, m, Diff([(k, DELETE, 0, ZERO32, ZERO32) for k in ks]))
    assert not m.acc
    ranges_checked(st, m, *whole(full), root=EMPTY)
    ranges_checked(st, full, *whole(full), back=1)
    ranges_checked(st, StateModel(oracle), *whole(full), back=2, root=EMPTY)
    st.close()


def test_refusals(ctx, oracle):
    rng = np.random.default_rng(3)
    st = ctx.resident_state()
    st.set_journal(2)
    m = StateModel(oracle)
    k = rkey(rng)
    apply_checked(st, m, Diff([(k, 0, 1, u32be(2), ZERO32)], [(0, rkey(rng), rval(rng))]))
    o, lim, ak = np.zeros(64, np.uint8), np.full(64, 0xff, np.uint8), np.frombuffer(k * 2, np.uint8).copy()
    mx = np.array([3, 3], np.uint32)

    def call(q, back=0, values=None):
        out = {f: np.full(256, 0xAA, np.uint8) for f, _ in gpu.RangeValues._fields_}
        v = values or gpu.RangeValues(*[out[f].ctypes.data for f, _ in gpu.RangeValues._fields_])
        root = np.full(32, 0xAA, np.uint8)
        rc = st.range_raw(q, back, v, root)
        if rc:
            assert (root == 0xAA).all() and all((x == 0xAA).all() for x in out.values()), "a refused range call wrote"
        return rc

    def req(n=2, ao=o, al=lim, am=mx, m_=2, sa=ak, so=o, sl=lim, sm=mx):
        p = lambda a: None if a is None else (a if isinstance(a, int) else a.ctypes.data)  # noqa: E731
        return gpu.RangeRequest(n, p(ao), p(al), p(am), m_, p(sa), p(so), p(sl), p(sm))

    assert call(req(), 1) == 0
    assert call(req(), 2) == E_INVALID                                    # back > journal_applies
    for f in ("ao", "al", "am", "sa", "so", "sl", "sm"):
        assert call(req(**{f: None})) == E_INVALID, f                     # a NULL array with a count
    assert call(req(n=(1 << 28) + 1, m_=0)) == E_INVALID                  # too many ranges
    assert call(req(n=0, m_=(1 << 28) + 1)) == E_INVALID
    big = np.array([1 << 31, 1 << 31], np.uint32)
    assert call(req(am=big)) == E_INVALID                                 # sum(max) >= 2^32
    assert call(req(sm=big)) == E_INVALID
    assert call(req(am=np.array([ALL, 0], np.uint32), sm=np.array([ALL, 0], np.uint32)), 1) == 0  # just below
    d = torch.from_numpy(o).cuda()
    torch.cuda.synchronize()
    assert call(req(ao=d.data_ptr())) == E_INVALID                        # device pointers: request
    dout = torch.zeros(256, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    v = gpu.RangeValues(*([None] * 2 + [dout.data_ptr()] + [None] * 8))
    assert call(req(), 0, v) == E_INVALID                                 # and outputs
    assert st.root() == m.root() and st.info()["journal_applies"] == 1
    st.close()


def test_a_range_call_changes_nothing(ctx, oracle):
    rng = np.random.default_rng(4)
    st, m, hist, ks = journaled(ctx, oracle, rng, n_blocks=2)
    root, info = st.root(), st.info()
    keep = ("n_accounts", "n_slots", "journal_applies", "journal_bytes")

    def unchanged():
        i = st.info()
        assert st.root() == root and all(i[f] == info[f] for f in keep)

    for back in (0, 2, 1, 0):
        ranges_checked(st, hist[len(hist) - 1 - back], *whole(m), back=back)
        unchanged()
    nd = block(rng, m, {ks[2]: (9, u32be(9), ZERO32)}, [(ks[3], rkey(rng), rval(rng))])
    want_nodes, want_off = st.witness(**nd.arrays())
    rc, size = st.witness_raw(st._diff(**nd.arrays()))
    assert rc == 0
    ranges_checked(st, hist[-2], *whole(m), back=1)
    nodes, off = np.zeros(max(size.nodes_bytes, 1), np.uint8), np.zeros(size.n_nodes + 1, np.uint64)
    assert st.witness_copy_raw(nodes, off) == 0
    assert nodes[:size.nodes_bytes].tobytes() == want_nodes.tobytes() and (off == want_off).all()
    ak = np.frombuffer(b"".join(ks[:5]), np.uint8).copy()
    want = st.prove(ak)
    rc, size = st.prove_raw(st._request(ak))
    assert rc == 0
    ranges_checked(st, m, *whole(m))
    r = dict(nodes=np.zeros(max(size.nodes_bytes, 1), np.uint8), node_off=np.zeros(size.n_nodes + 1, np.uint64),
             node_index=np.zeros(max(size.n_refs, 1), np.uint64), proof_first=np.zeros(6, np.uint64))
    p = gpu.Proofs(r["nodes"].ctypes.data, r["node_off"].ctypes.data, r["node_index"].ctypes.data, r["proof_first"].ctypes.data,
                   None, None, None, None, None, None, None)
    assert st.prove_copy_raw(p) == 0
    assert r["nodes"][:size.nodes_bytes].tobytes() == want["nodes"].tobytes() and (r["proof_first"] == want["proof_first"]).all()
    unchanged()
    st.close()


def test_at_size(ctx, oracle):
    """100k accounts, 1M slots, 64 journaled blocks: a whole-state dump at back 0 and 64 equals the model, with no Keccak;
    launches do not grow with the number of ranges or with back"""
    rng = np.random.default_rng(102)
    m, full = build_state(oracle, rng, 100_000, [(i * 100, 1000) for i in range(1000)])
    st = ctx.resident_state()
    assert st.apply(**full.arrays()) == m.root()
    m0 = m.copy()
    st.set_journal(64)
    keys = sorted(m.acc)
    for _ in range(64):
        touched = {keys[int(i)]: (int(rng.integers(0, 1 << 30)), u32be(rng.integers(1, 1 << 60)), rkey(rng))
                   for i in rng.choice(len(keys), 40, replace=False)}
        touched.update({rkey(rng): (1, u32be(1), ZERO32) for _ in range(5)})
        w = [(k, rkey(rng), rval(rng)) for k in list(touched)[:10]]
        d = block(rng, m, touched, w)
        st.apply(**d.arrays())
        m.apply(d)
    assert st.root() == m.root() and st.info()["journal_applies"] == 64
    rs = host.ResidentStateDB(ctx)
    rs.state.close()
    rs.state = st
    for back, h in ((0, m), (64, m0)):
        ctx.reset_stats()
        table = rs.dump(back=back, chunk=1 << 20)
        assert ctx.stats()["keccak_msgs"] == 0
        assert table.keys() == h.acc.keys()
        assert all(table[k] == (a.nonce, a.balance, a.code_hash, slots_of(h, k)) for k, a in h.acc.items())
    rich = [k for k in keys if m.acc[k].storage]
    launches = {}
    for back in (1, 64):
        for n in (10, 2000):
            sr = [(rich[i % len(rich)], ZERO_KEY, MAX_KEY, 20) for i in range(n)]
            ar = [(keys[i * 40], MAX_KEY, 20) for i in range(n)]
            ctx.reset_stats()
            st.range(ar, sr, back=back)
            s = ctx.stats()
            assert s["keccak_msgs"] == 0, s
            launches[back, n] = s["launches"]
    assert launches[1, 2000] < 2 * launches[1, 10] and launches[64, 2000] < 2 * launches[1, 2000], launches
    assert launches[64, 10] < 2 * launches[1, 10], launches
    st.close()


def test_storage_range_proof_host_layer(ctx, oracle, golden):
    """host.ResidentStateDB.storage_range / storage_range_proof on fixtures: the slots of the post state, and V accepts the
    boundary proofs with the origin present exactly when it is the first slot returned"""
    from test_gpu_resident_state_witness import fixture_touched
    g = golden("fixture_states.json.gz")
    seen = 0
    for t in g["tests"][:40]:
        old, touched, slots = fixture_touched(g["tables"][t["pre"]], g["tables"][t["post"]])
        rs = host.ResidentStateDB(ctx)
        if old:
            rs.apply(old)
        rs.apply(touched, slots)
        new = {a: s for a, s in old.items() if a not in touched}
        new.update({a: s for a, s in touched.items() if s is not None})
        for a, s in new.items():
            if not s.storage:
                continue
            want = sorted((oracle.keccak256(k.to_bytes(32, "big")), v) for k, v in s.storage.items())
            got, more = rs.storage_range(a, ZERO_KEY, MAX_KEY, len(want) + 1)
            assert got == want and not more
            p = rs.storage_range_proof(a, want[0][0], MAX_KEY, 1)
            assert p["slots"] == want[:1] and p["more"] == (len(want) > 1) and p["keys"] == [want[0][0]]
            pr = p["proof"]
            akey = oracle.keccak256(a)
            status, _ = verify(ctx, pr, [akey] + p["keys"])
            assert list(status) == [1, 1]
            seen += 1
        rs.close()
    assert seen
