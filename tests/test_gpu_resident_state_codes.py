"""Contract code kept beside the resident world state on the GPU (phant_gpu_resident_state_put_codes / _codes /
_prune_codes): hashes equal the oracle's Keccak and bytes round-trip; get_code equals the fixtures' code now and one block
back; prune keeps exactly what a reachable root names; witness_blob carries the codes read_payload_witness needs and gives
transition_root the header's root; every refusal changes nothing; no call disturbs the root, the journal or a held result;
and at size the lookups match a model at every `back` with launch counts that do not grow with the request."""
import ctypes as C

import numpy as np
import pytest
import torch

from phant_b200 import gpu
from phant_b200 import host
from test_gpu_resident_state_witness import fixture_touched

pytestmark = pytest.mark.gpu

E_INVALID = -1
EMPTY_CODE_HASH = host.EMPTY_CODE_HASH


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


def codes_of(table):
    return {bytes.fromhex(a["address"]): bytes.fromhex(a["code"]) for a in table}


def test_fixtures(ctx, oracle, golden):
    """pre loaded with its codes, the block applied with the post codes: get_code now and one block back, witness_blob into
    P and T, prune with and without the journal"""
    g = golden("fixture_states.json.gz")
    rng = np.random.default_rng(5)
    n = 0
    for t in g["tests"]:
        pre_t, post_t = g["tables"][t["pre"]], g["tables"][t["post"]]
        old, touched, slots = fixture_touched(pre_t, post_t)
        pre_code, post_code = codes_of(pre_t), codes_of(post_t)
        rs = host.ResidentStateDB(ctx)
        rs.set_journal(1)
        rs.put_codes(list(pre_code.values()))
        if old:
            assert rs.apply(old).hex() == t["pre_root"], t["name"]
        ghosts = [rng.bytes(20) for _ in range(3)]
        assert rs.get_code(list(pre_code) + ghosts) == {**pre_code, **{a: b"" for a in ghosts}}, t["name"]
        # the block's witness from the pre-state: complete for P, and T gives the header's root
        if touched:
            blob = rs.witness_blob(touched, slots)
            ps = host.read_payload_witness(ctx, bytes.fromhex(t["pre_root"]), blob, list(touched))
            assert ps.missing_code == [], t["name"]
            for a in touched:
                if a in old:
                    assert ps.account_status[a] == 1 and ps.accounts[a].code == old[a].code, t["name"]
            root, status = host.transition_root(ctx, bytes.fromhex(t["pre_root"]), blob, touched, slots)
            assert status == 1 and root.hex() == t["post_root"], t["name"]
        rs.put_codes(list(post_code.values()))
        assert rs.apply(touched, slots).hex() == t["post_root"], t["name"]
        everyone = list(dict.fromkeys(list(pre_code) + list(post_code) + ghosts))
        want_now = {a: post_code.get(a, b"") for a in everyone}
        want_before = {a: pre_code.get(a, b"") for a in everyone}
        assert rs.get_code(everyone) == want_now and rs.get_code(everyone, back=1) == want_before, t["name"]
        rs.prune_codes()
        assert rs.get_code(everyone) == want_now and rs.get_code(everyone, back=1) == want_before, t["name"]
        rs.set_journal(0)
        rs.prune_codes()
        post_set = {c for c in post_code.values() if c}
        info = rs.state.info()
        assert (info["n_codes"], info["code_bytes"]) == (len(post_set), sum(map(len, post_set))), t["name"]
        assert rs.get_code(everyone) == want_now, t["name"]
        rs.close()
        n += 1
    assert n == 84


def test_hashes_and_bytes(ctx, oracle):
    rng = np.random.default_rng(7)
    st = ctx.resident_state()
    lengths = [0, 1, 135, 136, 137, 272, 24_576, 1 << 20]
    codes = [rng.bytes(n) for n in lengths]
    hashes = st.put_codes(codes)
    assert [h.tobytes() for h in hashes] == [oracle.keccak256(c) for c in codes]
    assert hashes[0].tobytes() == EMPTY_CODE_HASH
    i = st.info()
    assert (i["n_codes"], i["code_bytes"]) == (7, sum(lengths))
    status, got = st.codes(hashes)
    assert list(status) == [1] * 8 and got == codes
    # duplicates within one call and across calls are stored once; the hashes still come back in order
    again = st.put_codes([codes[3], rng.bytes(40), codes[3], b"", codes[7]])
    assert st.info()["n_codes"] == 8 and st.info()["code_bytes"] == sum(lengths) + 40
    assert again[0].tobytes() == again[2].tobytes() == hashes[3].tobytes()
    # repeats, keccak(""), a hash that is not held
    ghost = rng.bytes(32)
    q = np.frombuffer(hashes[5].tobytes() + EMPTY_CODE_HASH + ghost + hashes[5].tobytes() + hashes[1].tobytes(), np.uint8)
    status, got = st.codes(q)
    assert list(status) == [1, 1, 2, 1, 1] and got == [codes[5], b"", b"", codes[5], codes[1]]
    # codes_cap too small: sizes written, bytes not
    stt, off = np.zeros(5, np.uint8), np.zeros(6, np.uint64)
    buf = np.full(1000, 0xAB, np.uint8)
    assert st.codes_raw(q, 5, stt, off, buf, 271) == 0
    assert list(stt) == [1, 1, 2, 1, 1] and list(off) == [0, 272, 272, 272, 544, 545] and (buf == 0xAB).all()
    assert st.codes_raw(q, 5, stt, off, buf, 545) == 0 and buf[:545].tobytes() == codes[5] + codes[5] + codes[1]
    assert (buf[545:] == 0xAB).all()
    st.close()


def snapshot(st):
    i = st.info()
    return st.root(), {k: v for k, v in i.items() if k != "device_bytes"}


def small_state(ctx, rng, n=200):
    st = ctx.resident_state()
    st.set_journal(4)
    codes = [rng.bytes(int(rng.integers(1, 500))) for _ in range(20)]
    hs = st.put_codes(codes)
    keys = np.frombuffer(rng.bytes(32 * n), np.uint8).reshape(n, 32)
    ch = np.stack([hs[i % 20] for i in range(n)])
    for b in range(3):
        st.apply(keys, np.full(n, b + 1, np.uint64), np.zeros((n, 32), np.uint8), np.roll(ch, b, axis=0))
    return st, keys, codes, hs


def test_refusals_change_nothing(ctx):
    rng = np.random.default_rng(8)
    st, _, codes, hs = small_state(ctx, rng)
    before = snapshot(st)
    q = np.concatenate(hs[:5]).reshape(-1)
    want = st.codes(q)
    data, off = gpu._csr_bytes([b"abc", b"defg"])
    out = np.zeros((2, 32), np.uint8)
    bad_off = np.array([0, 4, 3], np.uint64)
    huge = np.array([0, 1 << 32], np.uint64)
    d_data = torch.zeros(64, dtype=torch.uint8, device="cuda")
    d_off = torch.tensor([0, 3, 7], dtype=torch.int64, device="cuda")
    puts = [(None, off, 2, out), (data, None, 2, out), (data, bad_off, 2, out), (data, huge, 1, out), (data, off, 1 << 28, out),
            (d_data, off, 2, out), (data, d_off, 2, out), (data, off, 2, torch.zeros(64, dtype=torch.uint8, device="cuda"))]
    for args in puts:
        assert st.put_codes_raw(*args) == E_INVALID
        assert snapshot(st) == before
    stt, coff, buf = np.zeros(5, np.uint8), np.zeros(6, np.uint64), np.zeros(4096, np.uint8)
    d_q = torch.zeros(5 * 32, dtype=torch.uint8, device="cuda")
    looks = [(None, 5, stt, coff, buf, 4096), (q, 5, None, coff, buf, 4096), (q, 5, stt, None, buf, 4096), (q, 1 << 28, stt, coff, buf, 4096),
             (d_q, 5, stt, coff, buf, 4096), (q, 5, stt, coff, torch.zeros(4096, dtype=torch.uint8, device="cuda"), 4096)]
    for args in looks:
        assert st.codes_raw(*args) == E_INVALID
    status, got = st.codes(q)
    assert np.array_equal(status, want[0]) and got == want[1] and snapshot(st) == before
    st.close()


def test_nothing_else_changes(ctx):
    """root, the other info fields and the journal stay, and a held witness or proof result is still copied after each call"""
    rng = np.random.default_rng(9)
    st, keys, codes, hs = small_state(ctx, rng)
    root, info = snapshot(st)
    acct = lambda i: (keys[i:i + 1], np.array([9], np.uint64), np.zeros((1, 32), np.uint8), hs[0][None])  # noqa: E731
    calls = [lambda: st.put_codes([rng.bytes(77), codes[2]]), lambda: st.codes(np.concatenate(hs[:3])), lambda: st.prune_codes()]
    for call in calls:
        rc, size = st.witness_raw(gpu.ResidentState._diff(*acct(0), None, None, None, None))
        assert rc == 0 and size.n_nodes > 0
        call()
        nodes, off = np.zeros(max(size.nodes_bytes, 1), np.uint8), np.zeros(size.n_nodes + 1, np.uint64)
        assert st.witness_copy_raw(nodes, off) == 0
        q = gpu.ResidentState._request(keys[:3])
        rc, psize = st.prove_raw(q)
        assert rc == 0
        call()
        r = dict(nodes=np.zeros(max(psize.nodes_bytes, 1), np.uint8), node_off=np.zeros(psize.n_nodes + 1, np.uint64),
                 node_index=np.zeros(max(psize.n_refs, 1), np.uint64), proof_first=np.zeros(4, np.uint64))
        p = gpu.Proofs(*[gpu._ptr(r.get(f)) for f, _ in gpu.Proofs._fields_])
        assert st.prove_copy_raw(p) == 0
        r2, i2 = snapshot(st)
        assert r2 == root and {k: v for k, v in i2.items() if k not in ("n_codes", "code_bytes")} == \
            {k: v for k, v in info.items() if k not in ("n_codes", "code_bytes")}
    # the journal still reverts
    assert st.revert(2) != root
    st.close()


def block_arrays(keys, hashes, nonce):
    n = len(keys)
    return (np.stack(keys) if n else np.zeros((0, 32), np.uint8), np.full(n, nonce, np.uint64), np.zeros((n, 32), np.uint8),
            np.stack(hashes) if n else np.zeros((0, 32), np.uint8))


def test_at_size(ctx, oracle):
    """100k accounts, 20k distinct codes, 64 journaled blocks that create and destroy contracts"""
    rng = np.random.default_rng(11)
    st = ctx.resident_state()
    st.set_journal(64)
    pool = [rng.bytes(int(rng.integers(1, 600))) for _ in range(20_000)]
    ph = [h.tobytes() for h in st.put_codes(pool)]
    code_of = dict(zip(ph, pool))
    keys = [rng.bytes(32) for _ in range(100_000)]
    cur = {k: (ph[int(rng.integers(0, len(ph)))] if rng.random() < 0.4 else EMPTY_CODE_HASH) for k in keys}
    ks = list(cur)
    st.apply(*block_arrays([np.frombuffer(k, np.uint8) for k in ks], [np.frombuffer(cur[k], np.uint8) for k in ks], 1))
    undo = []  # per block: {key: code hash before, None = absent}
    live = list(keys)
    for b in range(64):
        fresh = [rng.bytes(int(rng.integers(1, 600))) for _ in range(20)]
        fh = [h.tobytes() for h in st.put_codes(fresh)]
        code_of.update(zip(fh, fresh))
        created = [rng.bytes(32) for _ in range(60)]
        changed = [live[int(i)] for i in rng.choice(len(live), 40, replace=False)]
        dead = set(changed[:15])
        changes = {k: fh[i % 20] for i, k in enumerate(created)} | {k: ph[int(rng.integers(0, len(ph)))] for k in changed[15:]}
        undo.append({k: cur.get(k) for k in list(changes) + list(dead)})
        flags = [0] * len(changes) + [gpu.ACCOUNT_DELETE] * len(dead)
        ak = [np.frombuffer(k, np.uint8) for k in list(changes) + list(dead)]
        hh = [np.frombuffer(h, np.uint8) for h in changes.values()] + [np.zeros(32, np.uint8)] * len(dead)
        st.apply(*block_arrays(ak, hh, b + 2), np.array(flags, np.uint8))
        cur.update(changes)
        for k in dead:
            del cur[k]
        live = [k for k in live if k not in dead] + created
    st.prune_codes()
    # every back: read the codeHash, look the code up, compare with the model walked back block by block
    probe = list(dict.fromkeys(keys + [k for u in undo for k in u]))
    pk = np.frombuffer(b"".join(probe), np.uint8)
    state = dict(cur)
    for back in range(65):
        if back:
            for k, h in undo[64 - back].items():
                if h is None:
                    state.pop(k, None)
                else:
                    state[k] = h
        r, _ = st.read(pk, back=back)
        hashes = np.where(r["account_status"][:, None] == 1, r["code_hash32"], np.frombuffer(EMPTY_CODE_HASH, np.uint8))
        status, got = st.codes(hashes)
        assert (status == 1).all(), back
        want = [code_of.get(state[k], b"") if k in state else b"" for k in probe]
        assert got == want, back
    # launches and Keccak messages do not depend on the request
    launches = []
    for q in (np.frombuffer(ph[3], np.uint8), np.frombuffer(b"".join(ph), np.uint8)):
        ctx.reset_stats()
        st.codes(q)
        s = ctx.stats()
        assert s["keccak_msgs"] == 0, s
        launches.append(s["launches"])
    one, keys1, _, _ = small_state(ctx, rng, 1)
    for s_ in (one, st):
        ctx.reset_stats()
        s_.prune_codes()
        s = ctx.stats()
        assert s["keccak_msgs"] == 0, s
        launches.append(s["launches"])
    assert launches[0] == launches[1] and launches[2] == launches[3], launches
    one.close()
    st.close()
