"""Account and slot reads from the resident world state (phant_gpu_resident_state_read) on the GPU, at the current root and
at every root the undo journal reaches: every value equals the Python model's snapshot of that block (storage roots
included), the returned root is that block's, and a read changes nothing -- not the root, the counts, the journal, nor a
witness or proof result the state holds."""
import numpy as np
import pytest
import torch

from phant_b200 import gpu
from phant_b200 import host
from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel, change_diff, hashed_table, load_diff
from test_gpu_resident_state import apply_checked, block, grow_account, rkey, rval, u32be
from test_gpu_resident_state_witness import fixture_touched
from test_gpu_transition_roots_at_size import build_state

pytestmark = pytest.mark.gpu

E_INVALID = -1
EMPTY = host.EMPTY_MPT_ROOT


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


def cat(keys):
    return np.frombuffer(b"".join(keys), np.uint8).copy() if keys else np.zeros(0, np.uint8)


def read(st, akeys, slots, back=0):
    """slots: [(account index, slot key)]"""
    sa = np.array([i for i, _ in slots], np.uint32) if slots else None
    return st.read(cat(akeys), sa, cat([k for _, k in slots]) if slots else None, back=back)


def read_checked(st, m, akeys, slots, back=0, root=None):
    """read at `back`; every value must be model m's, and the root `root` (default: m's)"""
    r, got = read(st, akeys, slots, back)
    assert got == (root if root is not None else m.root()), back
    for i, k in enumerate(akeys):
        a = m.acc.get(k)
        got_a = (int(r["account_status"][i]), int(r["nonce"][i]), r["balance32"][i].tobytes(), r["storage_root32"][i].tobytes(),
                 r["code_hash32"][i].tobytes())
        want = (2, 0, ZERO32, ZERO32, ZERO32) if a is None else (1, a.nonce, a.balance, m.storage_root(k), a.code_hash)
        assert got_a == want, (back, i, k.hex())
    for j, (i, sk) in enumerate(slots):
        a = m.acc.get(akeys[i])
        v = a.storage.get(sk, ZERO32) if a else ZERO32
        assert (int(r["slot_status"][j]), r["slot_vals32"][j].tobytes()) == ((1, v) if v != ZERO32 else (2, ZERO32)), (back, j)
    return r


def every_key(m, rng, n_absent=3):
    """every account and slot of m, absent accounts, and an absent slot per account"""
    akeys = sorted(m.acc) + [rkey(rng) for _ in range(n_absent)]
    slots = [(i, sk) for i, k in enumerate(akeys) if k in m.acc for sk in m.acc[k].storage]
    slots += [(i, rkey(rng)) for i in range(len(akeys))]
    return akeys, slots


def test_fixtures(ctx, oracle, golden):
    g = golden("fixture_states.json.gz")
    rng = np.random.default_rng(41)
    n = 0
    for t in g["tests"]:
        pre, post = hashed_table(oracle.keccak256, g["tables"][t["pre"]]), hashed_table(oracle.keccak256, g["tables"][t["post"]])
        st = ctx.resident_state()
        st.set_journal(1)
        m = StateModel(oracle)
        assert apply_checked(st, m, load_diff(pre)).hex() == t["pre_root"], t["name"]
        before = m.copy()
        akeys, slots = every_key(m, rng)
        read_checked(st, m, akeys, slots)
        apply_checked(st, m, change_diff(pre, post))
        assert m.root().hex() == t["post_root"]
        akeys, slots = every_key(m, rng)
        akeys += [k for k in before.acc if k not in m.acc]  # destroyed by the block
        slots += [(akeys.index(k), sk) for k in before.acc for sk in before.acc[k].storage]
        read_checked(st, m, akeys, slots, back=0)
        read_checked(st, before, akeys, slots, back=1)
        st.close()
        n += 1
    assert n == 84


def test_block_sequence_at_every_back(ctx, oracle):
    """the revert test's blocks at depth 16, read at every back after every block; then revert(3), another branch, and a
    shorter journal"""
    rng = np.random.default_rng(12)
    st = ctx.resident_state()
    st.set_journal(16)
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(6000)]
    big, doomed, reborn = keys[0], keys[1], keys[2]
    fields = lambda: (int(rng.integers(0, 1 << 20)), u32be(rng.integers(0, 1 << 60)), rkey(rng))  # noqa: E731
    hist = [(m.copy(), host.EMPTY_MPT_ROOT)]  # (model, root) after each block
    seen = {}  # big, doomed, reborn -> every slot key they held

    def step(d):
        root = apply_checked(st, m, d)
        hist.append((m.copy(), root))
        for k in (big, doomed, reborn):
            seen.setdefault(k, set()).update(m.acc[k].storage if k in m.acc else ())

    def check_all():
        pick = [big, doomed, reborn] + keys[3:203] + [rkey(rng) for _ in range(3)]
        slots = [(0, sk) for sk in sorted(seen.get(big, ()))[:3000]] + [(1, sk) for sk in sorted(seen.get(doomed, ()))]
        slots += [(2, sk) for sk in sorted(seen.get(reborn, ()))]
        slots += [(i, sk) for i, k in enumerate(pick[3:203], 3) for h, _ in hist[-3:] if k in h.acc for sk in h.acc[k].storage]
        slots += [(i, rkey(rng)) for i in range(len(pick))]
        n = st.info()["journal_applies"]
        for back in range(n + 1):
            h, root = hist[len(hist) - 1 - back]
            read_checked(st, h, pick, slots, back=back, root=root)

    writes = [(k, rkey(rng), rval(rng)) for k in keys[3:1003] for _ in range(int(rng.integers(1, 10)))]
    writes += grow_account(rng, m, big, 200) + grow_account(rng, m, doomed, 5000) + grow_account(rng, m, reborn, 300)
    step(block(rng, m, {k: fields() for k in keys}, writes))
    check_all()
    for target in (1000, 5000, 70000, 5000, 1000, 200):  # `big`: L 0 -> 1 -> 2 -> 3 and back
        touched = {keys[i]: fields() for i in rng.choice(np.arange(3, 6000), 30, replace=False)}
        w = grow_account(rng, m, big, target)
        small = [keys[i] for i in rng.choice(np.arange(3, 203), 30, replace=False)]
        w += [(k, list(m.acc[k].storage)[0], rval(rng)) for k in small if m.acc[k].storage]
        w += [(k, rkey(rng), ZERO32) for k in small[:5]]
        step(block(rng, m, touched, w))
        check_all()
    # `doomed` (5,000 slots) destroyed; `reborn` destroyed and created again in one apply
    step(block(rng, m, {doomed: (0, ZERO32, ZERO32), reborn: fields()}, [(reborn, rkey(rng), rval(rng)) for _ in range(40)],
               flags={doomed: DELETE, reborn: CLEAR}))
    check_all()
    step(block(rng, m, {}, []))  # an empty block is one apply too
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
    assert st.info()["journal_applies"] == 2
    check_all()
    with pytest.raises(gpu.PhantGpuError) as e:
        read(st, [big], [], back=3)
    assert e.value.code == E_INVALID
    st.close()


def test_crafted_premise_breaking_slot_keys(ctx, oracle):
    rng = np.random.default_rng(5)
    st = ctx.resident_state()
    st.set_journal(2)
    m = StateModel(oracle)
    a, b = rkey(rng), rkey(rng)
    f = (1, u32be(1), ZERO32)
    ka = [bytes([0xa0 | int(rng.integers(0, 16))]) + rkey(rng)[1:] for _ in range(300)]  # one first nibble
    kb = [b"\x5c" + rkey(rng)[1:] for _ in range(5000)]                                   # one first byte
    apply_checked(st, m, block(rng, m, {a: f, b: f}, [(a, k, rval(rng)) for k in ka] + [(b, k, rval(rng)) for k in kb]))
    before = m.copy()
    apply_checked(st, m, block(rng, m, {}, [(a, k, ZERO32) for k in ka[:100]] + [(b, k, rval(rng)) for k in kb[:100]]))
    near = [k[:31] + bytes([k[31] ^ 1]) for k in ka[:20] + kb[:20]]
    akeys = [a, b, rkey(rng)]
    slots = [(0, k) for k in ka + near] + [(1, k) for k in kb + near] + [(2, k) for k in ka[:5]]
    read_checked(st, m, akeys, slots)
    read_checked(st, before, akeys, slots, back=1)
    st.close()


def test_empty_state(ctx, oracle):
    rng = np.random.default_rng(1)
    st = ctx.resident_state()
    m = StateModel(oracle)
    read_checked(st, m, [rkey(rng) for _ in range(4)], [(0, rkey(rng)), (3, rkey(rng))], root=EMPTY)
    r, root = read(st, [], [])
    assert root == EMPTY and r["account_status"].size == 0
    st.set_journal(4)
    apply_checked(st, m, Diff([(rkey(rng), 0, 1, u32be(5), ZERO32)], [(0, rkey(rng), rval(rng))]))
    k = list(m.acc)[0]
    read_checked(st, StateModel(oracle), [k], [(0, list(m.acc[k].storage)[0])], back=1, root=EMPTY)
    st.close()


def test_duplicate_keys(ctx, oracle):
    rng = np.random.default_rng(2)
    st = ctx.resident_state()
    st.set_journal(1)
    m = StateModel(oracle)
    ks = [rkey(rng) for _ in range(3)]
    apply_checked(st, m, Diff([(k, 0, 7, u32be(9), rkey(rng)) for k in ks], [(i, rkey(rng), rval(rng)) for i in range(3) for _ in range(4)]))
    before = m.copy()
    apply_checked(st, m, Diff([(ks[0], CLEAR, 8, u32be(10), ZERO32)], [(0, rkey(rng), rval(rng))]))
    akeys = [ks[0], ks[1], ks[0], ks[0], rkey(rng)]
    slots = [(i, sk) for i in (0, 2, 3, 1) for h in (m, before) for sk in h.acc[akeys[i]].storage] * 2
    for back, h in ((0, m), (1, before)):
        r = read_checked(st, h, akeys, slots, back=back)
        assert (r["balance32"][0] == r["balance32"][2]).all() and (r["storage_root32"][0] == r["storage_root32"][3]).all()
    st.close()


def test_refusals(ctx, oracle):
    rng = np.random.default_rng(3)
    st = ctx.resident_state()
    st.set_journal(2)
    m = StateModel(oracle)
    k = rkey(rng)
    apply_checked(st, m, Diff([(k, 0, 1, u32be(2), ZERO32)], [(0, rkey(rng), rval(rng))]))
    ak = cat([k, rkey(rng)])
    sa, sk = np.array([0, 1], np.uint32), cat([rkey(rng), rkey(rng)])

    def call(q, back=0, values=None):
        out = {f: np.full(96, 0xAA, np.uint8) for f, _ in gpu.StateReadValues._fields_}
        v = values or gpu.StateReadValues(*[out[f].ctypes.data for f, _ in gpu.StateReadValues._fields_])
        root = np.full(32, 0xAA, np.uint8)
        rc = st.read_raw(q, back, v, root)
        if rc:
            assert (root == 0xAA).all() and all((o == 0xAA).all() for o in out.values()), "a refused read wrote"
        return rc

    ok = gpu.ProofRequest(2, ak.ctypes.data, 2, sa.ctypes.data, sk.ctypes.data)
    assert call(ok, 1) == 0
    assert call(ok, 2) == E_INVALID                                                  # back > journal_applies
    bad_sa = np.array([0, 2], np.uint32)
    assert call(gpu.ProofRequest(2, ak.ctypes.data, 2, bad_sa.ctypes.data, sk.ctypes.data)) == E_INVALID  # slot_account range
    assert call(gpu.ProofRequest(2, None, 0, None, None)) == E_INVALID              # NULL keys with a count
    assert call(gpu.ProofRequest(2, ak.ctypes.data, 2, None, sk.ctypes.data)) == E_INVALID
    assert call(gpu.ProofRequest(2, ak.ctypes.data, 2, sa.ctypes.data, None)) == E_INVALID
    dk = torch.from_numpy(ak).cuda()
    torch.cuda.synchronize()
    assert call(gpu.ProofRequest(2, dk.data_ptr(), 0, None, None)) == E_INVALID     # device pointers: keys
    dout = torch.zeros(96, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    v = gpu.StateReadValues(None, None, dout.data_ptr(), None, None, None, None)
    assert call(gpu.ProofRequest(2, ak.ctypes.data, 0, None, None), 0, v) == E_INVALID  # and outputs
    assert st.root() == m.root() and st.info()["journal_applies"] == 1
    st.close()


def test_a_read_changes_nothing(ctx, oracle):
    rng = np.random.default_rng(4)
    st = ctx.resident_state()
    st.set_journal(3)
    m = StateModel(oracle)
    ks = [rkey(rng) for _ in range(50)]
    apply_checked(st, m, Diff([(k, 0, 1, u32be(2), ZERO32) for k in ks], [(i, rkey(rng), rval(rng)) for i in range(50) for _ in range(3)]))
    before = m.copy()
    d = block(rng, m, {ks[0]: (5, u32be(6), ZERO32)}, [(ks[1], rkey(rng), rval(rng))])
    apply_checked(st, m, d)
    akeys, slots = every_key(m, rng)
    root, info = st.root(), st.info()

    def unchanged():
        i = st.info()
        assert st.root() == root
        assert (i["n_accounts"], i["n_slots"], i["journal_applies"], i["journal_bytes"]) == \
            (info["n_accounts"], info["n_slots"], info["journal_applies"], info["journal_bytes"])

    for back, h in ((0, m), (1, before), (0, m)):
        read_checked(st, h, akeys, slots, back=back)
        unchanged()
    # a held witness survives a read
    nd = block(rng, m, {ks[2]: (9, u32be(9), ZERO32)}, [(ks[3], rkey(rng), rval(rng))])
    want_nodes, want_off = st.witness(**nd.arrays())
    rc, size = st.witness_raw(st._diff(**nd.arrays()))
    assert rc == 0
    read_checked(st, before, akeys, slots, back=1)
    nodes, off = np.zeros(max(size.nodes_bytes, 1), np.uint8), np.zeros(size.n_nodes + 1, np.uint64)
    assert st.witness_copy_raw(nodes, off) == 0
    assert nodes[:size.nodes_bytes].tobytes() == want_nodes.tobytes() and (off == want_off).all()
    # so does a held proof result
    want = st.prove(cat(ks[:5]))
    rc, size = st.prove_raw(st._request(cat(ks[:5])))
    assert rc == 0
    read_checked(st, m, akeys, slots)
    r = dict(nodes=np.zeros(max(size.nodes_bytes, 1), np.uint8), node_off=np.zeros(size.n_nodes + 1, np.uint64),
             node_index=np.zeros(max(size.n_refs, 1), np.uint64), proof_first=np.zeros(6, np.uint64))
    p = gpu.Proofs(r["nodes"].ctypes.data, r["node_off"].ctypes.data, r["node_index"].ctypes.data, r["proof_first"].ctypes.data,
                   None, None, None, None, None, None, None)
    assert st.prove_copy_raw(p) == 0
    assert r["nodes"][:size.nodes_bytes].tobytes() == want["nodes"].tobytes() and (r["proof_first"] == want["proof_first"]).all()
    unchanged()
    st.close()


def test_at_size(ctx, oracle):
    """100k accounts, 1M slots, 64 journaled blocks: a 2,000-account read and a 10-account read make the same launches (at
    most 2) at back 0 and at back 64, with no Keccak; the values equal prove's for the same keys"""
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
        w = [(k, rkey(rng), rval(rng)) for k in list(touched)[:10]]
        d = block(rng, m, touched, w)
        st.apply(**d.arrays())
        m.apply(d)
    assert st.root() == m.root() and st.info()["journal_applies"] == 64
    rich = [k for k in keys if m0.acc[k].storage][:5]  # first, so that the 10-account read has slots too
    rest = [k for k in keys if k not in set(rich)]
    picks = rich + [rest[int(i)] for i in rng.choice(len(rest), 1990, replace=False)] + [rkey(rng) for _ in range(5)]
    slots = [(i, sk) for i, k in enumerate(picks) if k in m0.acc for sk in sorted(m0.acc[k].storage)[:50]]
    slots += [(i, sk) for i, k in enumerate(picks) if k in m.acc for sk in sorted(m.acc[k].storage)[-3:]]
    slots = list(dict.fromkeys(slots))
    ak = cat(picks)
    sa, sk = np.array([i for i, _ in slots], np.uint32), cat([s for _, s in slots])
    launches = {}
    for back in (0, 64):
        for n in (10, 2000):
            ctx.reset_stats()
            st.read(ak[:32 * n], sa[sa < n] if n < 2000 else sa, sk.reshape(-1, 32)[sa < n] if n < 2000 else sk, back=back)
            s = ctx.stats()
            assert s["keccak_msgs"] == 0, s
            launches[back, n] = s["launches"]
    assert set(launches.values()) == {2}, launches
    r = read_checked(st, m0, picks, slots, back=64, root=m0.root())
    now, _ = st.read(ak, sa, sk)
    p = st.prove(ak, sa, sk)
    assert (now["account_status"] == p["status"][:len(picks)]).all() and (now["slot_status"] == p["status"][len(picks):]).all()
    for f in ("nonce", "balance32", "storage_root32", "code_hash32", "slot_vals32"):
        assert (now[f] == p[f]).all(), f
    assert (r["account_status"] == 1).sum() == 1995
    assert st.root() == m.root()
    st.close()


def test_host_layer(ctx, oracle, golden):
    """host.ResidentStateDB.read on every fixture, now and one block back: the values of the pre and post states"""
    g = golden("fixture_states.json.gz")
    rng = np.random.default_rng(12)
    for t in g["tests"]:
        old, touched, slots = fixture_touched(g["tables"][t["pre"]], g["tables"][t["post"]])
        rs = host.ResidentStateDB(ctx)
        rs.set_journal(1)
        if old:
            assert rs.apply(old).hex() == t["pre_root"], t["name"]
        rs.apply(touched, slots)
        new = {a: s for a, s in old.items() if a not in touched}
        new.update({a: s for a, s in touched.items() if s is not None})
        ghost = bytes(rng.integers(0, 256, 20, dtype=np.uint8))
        req = {a: sorted(set(s.storage) | set(old[a].storage if a in old else ()))[:8] + [12345] for a, s in new.items()}
        req.update({a: sorted(s.storage)[:8] for a, s in old.items() if a not in new})
        req[ghost] = [1, 2]
        for back, state in ((0, new), (1, old)):
            got = rs.read(req, back=back)
            for a, ks in req.items():
                v, s = got[a], state.get(a)
                assert v["exists"] == (s is not None), t["name"]
                assert (v["nonce"], v["balance"], v["codeHash"]) == ((s.nonce, s.balance, oracle.keccak256(s.code)) if s else
                                                                    (0, 0, oracle.keccak256(b""))), t["name"]
                if s is None:
                    assert v["storageHash"] == EMPTY
                assert v["storage"] == {k: (s.storage.get(k, 0) if s else 0) for k in ks}, t["name"]
        proofs = rs.get_proofs({a: [] for a in new})
        got = rs.read({a: [] for a in new})
        assert all(got[a]["storageHash"] == proofs[a]["storageHash"] for a in new), t["name"]
        rs.close()
