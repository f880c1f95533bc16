"""Range proofs checked on the GPU (phant_gpu_verify_ranges): status and `more` equal the CPU statement
(tests/range_proof_oracle.py) on every honest answer and every mutation of the corpus, many ranges per call with different
roots and WHOLE ranges mixed in; every refusal leaves the outputs untouched; answers served by the resident world state are
accepted at size, and a dump verified chunk by chunk loads back into the same root."""
import ctypes as C

import numpy as np
import pytest
import torch

from phant_b200 import gpu
from phant_b200 import host
from range_proof_corpus import accept_cases, awkward_tries, fixture_tries, mutation_cases, random_tries, truth
from range_proof_oracle import verify_range
from resident_range_model import MAX_KEY, ZERO_KEY
from resident_state_model import Diff
from test_gpu_resident_state_ranges import journaled, slots_of

pytestmark = pytest.mark.gpu

E_INVALID = -1


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


def one_call(ctx, cases):
    """cases [(root, origin, entries, nodes, whole)] in ONE call over the union of their node sets -> (status, more) lists"""
    nodes = list(dict.fromkeys(n for c in cases for n in c[3]))
    got = host.verify_ranges(ctx, [(r, o, e, w) for r, o, e, _, w in cases], nodes)
    return nodes, got


def check_against_statement(oracle, ctx, cases):
    nodes, got = one_call(ctx, cases)
    nodes = {oracle.keccak256(n): n for n in nodes}
    for (root, origin, ents, _, whole), g in zip(cases, got):
        assert g == verify_range(oracle.keccak256, nodes, root, origin, ents, whole), (origin.hex(), len(ents), whole)
    return got


def test_corpus_honest_answers(ctx, oracle, golden):
    rng = np.random.default_rng(3)
    tries = fixture_tries(oracle, golden) + random_tries(oracle) + awkward_tries(oracle)
    cases, wants = [], []
    for t in tries:
        for origin, ents, nodes, whole, more in accept_cases(t, limit=48, rng=rng):
            cases.append((t.root, origin, ents, nodes, whole))
            wants.append((1, more))
    order = rng.permutation(len(cases))
    cases, wants = [cases[i] for i in order], [wants[i] for i in order]
    assert len(cases) > 4000
    for a in range(0, len(cases), 1500):
        got = check_against_statement(oracle, ctx, cases[a:a + 1500])
        assert got == wants[a:a + 1500]


def test_corpus_mutations(ctx, oracle):
    """one call per kind of mutation, over tries that share no node: the GPU equals the statement, and only drop-last (a
    shorter honest answer) may be accepted -- with more set"""
    rng = np.random.default_rng(5)
    by_name = {}
    for t in random_tries(oracle) + awkward_tries(oracle):
        for name, root, origin, ents, nodes, whole in mutation_cases(t, rng):
            by_name.setdefault(name, []).append((t, (root, origin, ents, nodes, whole)))
    assert len(by_name) > 20
    for name, items in by_name.items():
        got = check_against_statement(oracle, ctx, [c for _, c in items])
        for (t, (root, origin, ents, _, whole)), (st, more) in zip(items, got):
            if name == "drop-last" and root == t.root and truth(t, origin, ents, whole)[0]:
                assert st != 1 or more, name
            else:
                assert st in (0, 3), (name, t.name)


def test_mixed_roots_and_whole_in_one_call(ctx, oracle):
    """honest answers, WHOLE ranges and mutations of several tries interleaved in one call"""
    rng = np.random.default_rng(6)
    cases = []
    for t in random_tries(oracle) + awkward_tries(oracle):
        for origin, ents, nodes, whole, _ in accept_cases(t, counts=(2, None), limit=6, rng=rng):
            cases.append((t.root, origin, ents, nodes, whole))
        cases += [c[1:] for c in mutation_cases(t, rng) if not c[0].startswith(("drop-node", "node-byte"))]
    order = rng.permutation(len(cases))
    check_against_statement(oracle, ctx, [cases[i] for i in order])


def _struct(n=3):
    """a valid 3-range call (no nodes, WHOLE ranges of the empty trie and a two-entry trie) and the arrays it points at"""
    keys = np.frombuffer(bytes(31) + b"\x01" + bytes(31) + b"\x02", np.uint8).copy()
    vals, voff = np.frombuffer(b"\x01\x02", np.uint8).copy(), np.array([0, 1, 2], np.uint64)
    roots = np.frombuffer(host.EMPTY_MPT_ROOT * n, np.uint8).copy()
    origins = np.zeros(32 * n, np.uint8)
    first = np.array([0] * n + [2], np.uint64)
    flags = np.ones(n, np.uint8)
    noff = np.zeros(1, np.uint64)
    nodes = np.zeros(1, np.uint8)
    keep = dict(keys=keys, vals=vals, voff=voff, roots=roots, origins=origins, first=first, flags=flags, noff=noff, nodes=nodes)
    s = gpu.RangeProofs(0, nodes.ctypes.data, noff.ctypes.data, 0, n, roots.ctypes.data, origins.ctypes.data, flags.ctypes.data,
                        first.ctypes.data, keys.ctypes.data, vals.ctypes.data, voff.ctypes.data)
    return s, keep


def test_refusals(ctx):
    status, more = np.full(3, 0xAA, np.uint8), np.full(3, 0xAA, np.uint8)
    s, k = _struct()
    assert ctx.verify_ranges_raw(s, status, more) == 0
    assert list(status) == [1, 1, 0] and list(more) == [0, 0, 0]  # the last range holds both entries, which are not the empty trie

    def refused(mutate, *extra):
        s, k = _struct()
        mutate(s, k)
        st, mo = np.full(3, 0xAA, np.uint8), np.full(3, 0xAA, np.uint8)
        ctx.reset_stats()
        assert ctx.verify_ranges_raw(s, st, mo) == E_INVALID
        assert (st == 0xAA).all() and (mo == 0xAA).all()
        assert ctx.stats()["launches"] == 0

    refused(lambda s, k: setattr(s, "roots32", None))
    refused(lambda s, k: setattr(s, "origin32", None))
    refused(lambda s, k: setattr(s, "entry_first", None))
    refused(lambda s, k: setattr(s, "keys32", None))
    refused(lambda s, k: setattr(s, "val_off", None))
    refused(lambda s, k: setattr(s, "vals", None))
    refused(lambda s, k: (s.__setattr__("n_nodes", 1), s.__setattr__("node_off", None)))
    refused(lambda s, k: k["first"].__setitem__(0, 1))
    refused(lambda s, k: k["first"].__setitem__(1, 2))          # 2, 0, 2: not monotone
    refused(lambda s, k: k["voff"].__setitem__(1, 3))
    refused(lambda s, k: k["flags"].__setitem__(1, 2))
    refused(lambda s, k: setattr(s, "n_nodes", (1 << 30) + 1))
    refused(lambda s, k: setattr(s, "n_ranges", (1 << 30) + 1))
    refused(lambda s, k: k["first"].__setitem__(3, (1 << 30) + 1))
    refused(lambda s, k: k["voff"].__setitem__(2, 1 << 33))
    node_off = np.array([0, 5, 2], np.uint64)
    refused(lambda s, k: (s.__setattr__("n_nodes", 2), s.__setattr__("node_off", node_off.ctypes.data)))
    d = torch.zeros(64, dtype=torch.uint8, device="cuda")
    refused(lambda s, k: setattr(s, "keys32", d.data_ptr()))
    s, k = _struct()
    s.n_ranges = 0
    st = np.full(3, 0xAA, np.uint8)
    assert ctx.verify_ranges_raw(s, st, None) == 0 and (st == 0xAA).all()
    s, k = _struct()
    st = np.full(3, 0xAA, np.uint8)
    s.range_flags = None
    assert ctx.verify_ranges_raw(s, st, None) == 0 and st[0] == 1  # flags NULL: all 0, an empty answer of the empty trie


def _served(ctx, st, akeys, rich, n_acc, n_st, per):
    """n_acc account ranges and n_st partial storage ranges served by range + prove, as one set of ranges and one node set,
    with the range call's `more` for each"""
    root = st.root()
    rng = np.random.default_rng(n_acc + n_st)
    aor = [akeys[int(i)] for i in rng.choice(len(akeys), n_acc, replace=False)]
    sac = [rich[int(i) % len(rich)] for i in rng.choice(len(rich), n_st, replace=n_st > len(rich))]
    r, _ = st.range([(o, MAX_KEY, per) for o in aor], [(a, ZERO_KEY, MAX_KEY, per) for a in sac])
    reads, _ = st.read(np.frombuffer(b"".join(sac), np.uint8)) if sac else ({}, None)
    ranges, more, prove_keys, slot_acc, slot_keys = [], [], [], [], []
    af, sf = r["account_first"], r["slot_first"]
    for i, o in enumerate(aor):
        a, b = int(af[i]), int(af[i + 1])
        ents = [(r["account_keys32"][e].tobytes(), host._account_value(dict(
            nonce=int(r["nonce"][e]), balance=int.from_bytes(r["balance32"][e].tobytes(), "big"),
            storageHash=r["storage_root32"][e].tobytes(), codeHash=r["code_hash32"][e].tobytes()))) for e in range(a, b)]
        ranges.append((root, o, ents, False))
        more.append(bool(r["account_more"][i]))
        prove_keys += [o] + [ents[-1][0]] * bool(ents)
    for j, ak in enumerate(sac):
        a, b = int(sf[j]), int(sf[j + 1])
        ents = [(r["slot_keys32"][e].tobytes(), host._rlp_str(r["slot_vals32"][e].tobytes().lstrip(b"\x00"))) for e in range(a, b)]
        ranges.append((reads["storage_root32"][j].tobytes(), ZERO_KEY, ents, False))
        more.append(bool(r["slot_more"][j]))
        slot_acc += [len(prove_keys) + j] * 2
        slot_keys += [ZERO_KEY, ents[-1][0]]
    allk = prove_keys + sac
    p = st.prove(np.frombuffer(b"".join(allk), np.uint8), np.array(slot_acc, np.uint32) if slot_acc else None,
                 np.frombuffer(b"".join(slot_keys), np.uint8) if slot_keys else None)
    return ranges, more, p


def test_resident_state_at_size(ctx, oracle):
    """100k accounts and 1M slots: 256 served ranges in one call are all accepted, each with the range call's `more`, and
    the call makes fewer than twice the launches of a one-range call"""
    rng = np.random.default_rng(104)
    n = 100_000
    keys = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    d = Diff([(keys[i].tobytes(), 0, i, (i + 1).to_bytes(32, "big"), bytes(32)) for i in range(n)])
    for ai in range(0, 100_000, 100):
        sk = rng.integers(0, 256, (1000, 32), dtype=np.uint8)
        d.slots += [(ai, sk[j].tobytes(), (j + 1).to_bytes(32, "big")) for j in range(1000)]
    st = ctx.resident_state()
    st.apply(**d.arrays())
    akeys = [keys[i].tobytes() for i in range(n)]
    rich = [akeys[i] for i in range(0, n, 100)]
    launches = {}
    for n_acc, n_st in ((1, 0), (192, 64)):
        ranges, more, p = _served(ctx, st, akeys, rich, n_acc, n_st, 300)
        ctx.reset_stats()
        got = host.verify_ranges(ctx, ranges, p)
        launches[n_acc + n_st] = ctx.stats()["launches"]
        assert got == [(1, m) for m in more]
        assert any(more) or n_acc == 1
    assert launches[256] < 2 * launches[1], launches
    st.close()


def _storage_answer(st, akey, origin, chunk):
    """storage_range_proof for a hashed account key: the slots from origin and the boundary proofs in its storage trie"""
    r, _ = st.range(storage_ranges=[(akey, origin, MAX_KEY, chunk)])
    slots = [(r["slot_keys32"][e].tobytes(), int.from_bytes(r["slot_vals32"][e].tobytes(), "big")) for e in range(int(r["slot_first"][1]))]
    keys = list(dict.fromkeys([origin] + [s[0] for s in slots[-1:]]))
    proof = st.prove(np.frombuffer(akey, np.uint8), np.zeros(len(keys), np.uint32), np.frombuffer(b"".join(keys), np.uint8))
    return slots, bool(r["slot_more"][0]), proof


def test_round_trip(ctx, oracle):
    """a journaled state dumped through account_range_proof and storage ranges with proofs, in chunks; every answer verified;
    the verified entries loaded into a fresh state with one apply give the source's root and storage roots; the same answers
    against the root one block older are rejected"""
    rng = np.random.default_rng(12)
    st, m, hist, _ = journaled(ctx, oracle, rng, n_blocks=3)
    rs = host.ResidentStateDB(ctx)
    rs.state.close()
    rs.state = st
    root, old_root = st.root(), hist[-2].root()
    assert root == m.root() and old_root != root
    accounts, origin, answers = [], bytes(32), 0
    while True:
        p = rs.account_range_proof(origin, MAX_KEY, 37)
        assert host.verify_account_range(ctx, root, origin, p["accounts"], p["proof"]) == (True, p["more"])
        assert not host.verify_account_range(ctx, old_root, origin, p["accounts"], p["proof"])[0]
        accounts += p["accounts"]
        answers += 1
        if not p["more"]:
            break
        origin = host._next_key(p["accounts"][-1][0])
    assert answers > 5 and [k for k, _ in accounts] == sorted(m.acc)
    slots = {}
    old = {k: hist[-2].storage_root(k) for k in m.acc}
    for k, a in accounts:
        if a["storageHash"] == host.EMPTY_MPT_ROOT:
            continue
        o, got = bytes(32), []
        while True:
            sl, more, proof = _storage_answer(st, k, o, 23)
            whole = o == bytes(32) and not more
            res = host.verify_storage_ranges(ctx, [(a["storageHash"], o, sl)], proof, last_is_partial=not whole)
            assert res == [(True, more)]
            if old[k] != a["storageHash"]:
                assert not host.verify_storage_ranges(ctx, [(old[k], o, sl)], proof, last_is_partial=not whole)[0][0]
            got += sl
            if not more:
                break
            o = host._next_key(sl[-1][0])
        slots[k] = got
    assert slots and all(dict(v) == {sk: int.from_bytes(x, "big") for sk, x in slots_of(m, k).items()} for k, v in slots.items())
    d = Diff([(k, 0, a["nonce"], a["balance"].to_bytes(32, "big"), a["codeHash"]) for k, a in accounts])
    idx = {k: i for i, (k, _) in enumerate(accounts)}
    d.slots = [(idx[k], sk, v.to_bytes(32, "big")) for k, v_ in slots.items() for sk, v in v_]
    fresh = ctx.resident_state()
    got, sroots = fresh.apply(**d.arrays(), storage_roots=True)
    assert got == root
    assert all(sroots[i].tobytes() == a["storageHash"] for i, (_, a) in enumerate(accounts))
    fresh.close()
    rs.close()


def test_snap_storage_shape(ctx, oracle):
    """verify_storage_ranges: whole storage tries then one partial range, in one call, as GetStorageRanges answers"""
    rng = np.random.default_rng(13)
    st, m, _, _ = journaled(ctx, oracle, rng, n_blocks=1)
    rich = [k for k in sorted(m.acc) if slots_of(m, k)]
    ranges = []
    for k in rich[:5]:
        sl, more, _ = _storage_answer(st, k, bytes(32), 1 << 20)
        assert not more
        ranges.append((m.storage_root(k), bytes(32), sl))
    big = max(rich, key=lambda k: len(slots_of(m, k)))
    sl, more, proof = _storage_answer(st, big, bytes(32), 7)
    assert more
    ranges.append((m.storage_root(big), bytes(32), sl))
    assert host.verify_storage_ranges(ctx, ranges, proof, last_is_partial=True) == [(True, False)] * 5 + [(True, True)]
    bad = ranges[:1] + [(ranges[1][0], bytes(32), ranges[1][2][1:])] + ranges[2:]
    assert [ok for ok, _ in host.verify_storage_ranges(ctx, bad, proof, last_is_partial=True)] == [True, False, True, True, True, True]
    assert C.sizeof(gpu.RangeProofs) == 12 * 8
