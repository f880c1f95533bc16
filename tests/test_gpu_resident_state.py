"""The resident world state (phant_gpu_resident_state_*) on the GPU: after every apply the state root and every listed
account's storage root equal the Python model (tests/resident_state_model.py), which the CPU tests pin to the fixtures."""
import numpy as np
import pytest

from phant_b200 import gpu
from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel, change_diff, hashed_table, load_diff

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


def apply_checked(st, model, d):
    """apply d to the GPU state and the model; the root and the storage roots must agree"""
    root, sroots = st.apply(**d.arrays(), storage_roots=True)
    model.apply(d)
    assert root == model.root()
    for i, a in enumerate(d.accounts):
        assert sroots[i].tobytes() == model.storage_root(a[0]), i
    assert st.root() == root
    return root


def u32be(x):
    return int(x).to_bytes(32, "big")


def rkey(rng):
    return bytes(rng.integers(0, 256, 32, dtype=np.uint8))


def rval(rng):
    return bytes(rng.integers(0, 256, int(rng.integers(1, 33)), dtype=np.uint8)).rjust(32, b"\x00").replace(ZERO32, u32be(1))


def test_fixtures_load_pre_then_apply_only_the_changes(ctx, oracle, golden):
    g = golden("fixture_states.json.gz")
    n = 0
    for t in g["tests"]:
        pre, post = hashed_table(oracle.keccak256, g["tables"][t["pre"]]), hashed_table(oracle.keccak256, g["tables"][t["post"]])
        st = ctx.resident_state()
        m = StateModel(oracle)
        assert apply_checked(st, m, load_diff(pre)).hex() == t["pre_root"], t["name"]
        tab = g["tables"][t["pre"]]
        assert ctx.state_root(*state_root_args(tab)).hex() == t["pre_root"]
        assert apply_checked(st, m, change_diff(pre, post)).hex() == t["post_root"], t["name"]
        info = st.info()
        assert info["n_accounts"] == len(post)
        assert info["n_slots"] == sum(1 for v in post.values() for x in v[3].values() if x != ZERO32)
        st.close()
        n += 1
    assert n == 84


def state_root_args(tab):
    n = len(tab)
    addr = np.frombuffer(b"".join(bytes.fromhex(a["address"]) for a in tab), np.uint8)
    nonce = np.array([a["nonce"] for a in tab], np.uint64)
    bal = np.frombuffer(b"".join(bytes.fromhex(a["balance"]) for a in tab), np.uint8)
    codes = [bytes.fromhex(a["code"]) for a in tab]
    code = np.frombuffer(b"".join(codes) or b"\x00", np.uint8)
    coff = np.concatenate([[0], np.cumsum([len(c) for c in codes])]).astype(np.uint64)
    sk = [bytes.fromhex(k) for a in tab for k in a["storage"]]
    sv = [bytes.fromhex(v) for a in tab for v in a["storage"].values()]
    soff = np.concatenate([[0], np.cumsum([len(a["storage"]) for a in tab])]).astype(np.uint64)
    return (n, addr, nonce, bal, code, coff, np.frombuffer(b"".join(sk) or b"\x00", np.uint8), np.frombuffer(b"".join(sv) or b"\x00", np.uint8), soff)


def grow_account(rng, m, key, target):
    """slot writes that take account `key` of the model to `target` live slots"""
    have = list(m.acc[key].storage) if key in m.acc else []
    if target >= len(have):
        return [(key, rkey(rng), rval(rng)) for _ in range(target - len(have))]
    drop = rng.choice(len(have), len(have) - target, replace=False)
    return [(key, have[i], ZERO32) for i in drop]


def block(rng, m, acc_fields, slot_writes, flags=None):
    """a Diff listing every account in acc_fields (key -> (nonce, balance, code)) plus the accounts the slot writes need"""
    flags = flags or {}
    order, idx = [], {}
    for k in list(acc_fields) + [w[0] for w in slot_writes]:
        if k not in idx:
            idx[k] = len(order)
            order.append(k)
    accounts = []
    for k in order:
        if k in acc_fields:
            f = acc_fields[k]
        else:
            a = m.acc[k]
            f = (a.nonce, a.balance, a.code_hash)
        accounts.append((k, flags.get(k, 0), f[0], f[1], f[2]))
    perm = rng.permutation(len(slot_writes))
    return Diff(accounts, [(idx[slot_writes[i][0]], slot_writes[i][1], slot_writes[i][2]) for i in perm])


def test_block_sequence_with_depth_changes_destroys_and_recreation(ctx, oracle):
    rng = np.random.default_rng(11)
    st = ctx.resident_state()
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(20000)]
    big, doomed, reborn = keys[0], keys[1], keys[2]
    fields = lambda: (int(rng.integers(0, 1 << 20)), u32be(rng.integers(0, 1 << 60)), rkey(rng))  # noqa: E731
    # block 0: load; 2,000 small storage tries, `big` with 200 slots (L 0), `doomed` with 5,000 (L 2), `reborn` with 300
    writes = [(k, rkey(rng), rval(rng)) for k in keys[3:2003] for _ in range(int(rng.integers(1, 30)))]
    writes += grow_account(rng, m, big, 200) + grow_account(rng, m, doomed, 5000) + grow_account(rng, m, reborn, 300)
    writes += [(keys[5000], rkey(rng), ZERO32)]  # an absent slot written as zero
    apply_checked(st, m, block(rng, m, {k: fields() for k in keys}, writes))
    assert st.info()["n_accounts"] == 20000
    # `big`: 200 -> 1,000 -> 5,000 -> 70,000 slots (L 0 -> 1 -> 2 -> 3), then back down
    for target in (1000, 5000, 70000, 5000, 1000, 200):
        touched = {keys[i]: fields() for i in rng.choice(np.arange(3, 20000), 50, replace=False)}
        w = grow_account(rng, m, big, target)
        small = [keys[i] for i in rng.choice(np.arange(3, 2003), 40, replace=False)]
        w += [(k, list(m.acc[k].storage)[0], rval(rng)) for k in small if m.acc[k].storage]  # slot changes, fields unchanged
        w += [(k, rkey(rng), ZERO32) for k in small[:5]]                                     # absent slots written as zero
        apply_checked(st, m, block(rng, m, touched, w))                                       # `touched`: no slot change
    assert len(m.acc[big].storage) == 200
    # `doomed` destroyed while it holds 5,000 slots; `reborn` destroyed and re-created in the same apply
    d = block(rng, m, {doomed: (0, ZERO32, ZERO32), reborn: fields()}, [(reborn, rkey(rng), rval(rng)) for _ in range(40)],
              flags={doomed: DELETE, reborn: CLEAR})
    apply_checked(st, m, d)
    assert doomed not in m.acc and len(m.acc[reborn].storage) == 40
    # values only: existing accounts, existing slots, new non-zero values
    live = [k for k in keys[3:2003] if m.acc[k].storage]
    w = [(k, sk, rval(rng)) for k in live[:500] for sk in list(m.acc[k].storage)[:3]] + [(big, sk, rval(rng)) for sk in list(m.acc[big].storage)[:50]]
    before = st.info()["n_slots"]
    apply_checked(st, m, block(rng, m, {}, w))
    assert st.info()["n_slots"] == before
    # deletes of whole storage tries and of absent accounts
    ghost = rkey(rng)
    apply_checked(st, m, block(rng, m, {keys[7]: (0, ZERO32, ZERO32), ghost: (0, ZERO32, ZERO32)}, [], flags={keys[7]: DELETE, ghost: DELETE}))
    assert keys[7] not in m.acc and ghost not in m.acc
    st.close()


def test_crafted_slot_keys_break_the_dense_top_premise(ctx, oracle):
    rng = np.random.default_rng(3)
    st = ctx.resident_state()
    m = StateModel(oracle)
    a, b, c = rkey(rng), rkey(rng), rkey(rng)
    one = lambda: bytes([int(rng.integers(1, 0x80))]).rjust(32, b"\x00")  # noqa: E731
    # a: 300 keys under one first nibble (L 1 -> the root has one child); b: 5,000 keys under one first byte (L 2 -> twice
    # lowered); c: long shared prefixes and pairs that differ in the last nibble only, 1-byte values (embedded leaves)
    ka = [bytes([0xa0 | int(rng.integers(0, 16))]) + rkey(rng)[1:] for _ in range(300)]
    kb = [b"\x5c" + rkey(rng)[1:] for _ in range(5000)]
    kc = []
    for i in range(150):
        base = b"\x77" * 28 + bytes([i]) + rkey(rng)[:2]
        kc += [base + bytes([0x10]), base + bytes([0x11])]
    w = [(a, k, one()) for k in ka] + [(b, k, one()) for k in kb] + [(c, k, one()) for k in kc]
    apply_checked(st, m, block(rng, m, {a: (1, u32be(1), ZERO32), b: (2, u32be(2), ZERO32), c: (3, u32be(3), ZERO32)}, w))
    for _ in range(3):  # incremental changes on top of the lowered depths, and a few slots outside the crafted prefixes
        w = [(a, ka[i], one()) for i in rng.choice(300, 20, replace=False)] + [(b, kb[i], ZERO32) for i in rng.choice(5000, 30, replace=False)]
        w += [(b, rkey(rng), one()) for _ in range(10)] + [(c, kc[i], ZERO32) for i in rng.choice(300, 10, replace=False)]
        w = list({(x[0], x[1]): x for x in w}.values())
        apply_checked(st, m, block(rng, m, {}, w))
    st.close()


def test_refused_applies_leave_the_state_unchanged(ctx, oracle):
    rng = np.random.default_rng(8)
    for loaded in (False, True):
        st = ctx.resident_state()
        m = StateModel(oracle)
        if loaded:
            ks = [rkey(rng) for _ in range(300)]
            apply_checked(st, m, block(rng, m, {k: (1, u32be(5), ZERO32) for k in ks}, [(k, rkey(rng), rval(rng)) for k in ks for _ in range(3)]))
        k1, k2, s1 = rkey(rng), rkey(rng), rkey(rng)
        f = (1, u32be(9), ZERO32)
        bad = [Diff([(k1,) + (0,) + f, (k1,) + (0,) + f]),                                   # the same account twice
               Diff([(k1, 0) + f], [(0, s1, u32be(1)), (0, s1, u32be(2))]),                   # the same slot twice
               Diff([(k1, 0) + f], [(1, s1, u32be(1))]),                                      # slot_account out of range
               Diff([(k1, DELETE) + f, (k2, 0) + f], [(0, s1, u32be(1))]),                    # a slot of a deleted account
               Diff([(k1, 4) + f])]                                                           # unknown flag bits
        for d in bad:
            root = st.root()
            with pytest.raises(gpu.PhantGpuError) as e:
                st.apply(**d.arrays())
            assert e.value.code == -1
            assert st.root() == root
        import torch
        dev_keys = torch.zeros(32, dtype=torch.uint8, device="cuda")
        a = Diff([(k1, 0) + f]).arrays()
        raw = gpu.StateDiff(1, dev_keys.data_ptr(), None, a["nonce"].ctypes.data, a["balance32"].ctypes.data, a["code_hash32"].ctypes.data, 0,
                            None, None, None)
        root = st.root()
        assert st.apply_raw(raw) == -1 and st.root() == root
        apply_checked(st, m, Diff([(k1, 0) + f, (k2, 0) + f], [(0, s1, u32be(7))]))
        st.close()


def test_incremental_work_from_the_stats(ctx, oracle):
    rng = np.random.default_rng(21)
    st = ctx.resident_state()
    m = StateModel(oracle)
    big, other = rkey(rng), rkey(rng)
    n = 1_000_000
    sk = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    sv = np.zeros((n, 32), np.uint8)
    sv[:, 31] = 1 + rng.integers(0, 255, n)
    d = Diff([(big, 0, 1, u32be(1), ZERO32), (other, 0, 1, u32be(1), ZERO32)])
    a = d.arrays()
    a.update(slot_account=np.zeros(n, np.uint32), slot_keys32=sk.reshape(-1), slot_vals32=sv.reshape(-1))
    st.apply(**a)
    m.apply(d)
    m.acc[big].storage = {sk[i].tobytes(): sv[i].tobytes() for i in range(n)}
    assert st.root() == m.root()
    # one slot of the 1,000,000-slot account (L 3): one bucket of ~244 slots and three dense nodes, not a rebuild
    ctx.reset_stats()
    apply_checked(st, m, Diff([(big, 0, 1, u32be(1), ZERO32)], [(0, sk[5].tobytes(), u32be(99))]))
    assert ctx.stats()["keccak_msgs"] < 2000
    # touching another account does not rehash the big account's storage
    ctx.reset_stats()
    apply_checked(st, m, Diff([(other, 0, 2, u32be(2), ZERO32)], [(0, rkey(rng), u32be(3))]))
    assert ctx.stats()["keccak_msgs"] < 200
    # launches do not grow with the number of touched accounts (same L mix: L 0 storage tries)
    ks = [rkey(rng) for _ in range(2000)]
    apply_checked(st, m, block(rng, m, {k: (1, u32be(1), ZERO32) for k in ks}, [(k, rkey(rng), rval(rng)) for k in ks for _ in range(3)]))
    launches = []
    for cnt in (10, 2000):
        ctx.reset_stats()
        apply_checked(st, m, block(rng, m, {k: (2, u32be(cnt), ZERO32) for k in ks[:cnt]}, [(k, rkey(rng), rval(rng)) for k in ks[:cnt]]))
        launches.append(ctx.stats()["launches"])
    assert launches[1] < 2 * launches[0], launches
    st.close()


def test_device_memory_stays_bounded_by_the_live_contents(ctx, oracle):
    rng = np.random.default_rng(4)
    st = ctx.resident_state()
    m = StateModel(oracle)
    ks = [rkey(rng) for _ in range(5000)]
    slots = {k: [rkey(rng), rkey(rng)] for k in ks}
    after_second = None
    for it in range(100):
        d = Diff([(k, 0, it, u32be(int(rng.integers(1, 1 << 62))), ZERO32) for k in ks],
                 [(i, s, rval(rng)) for i, k in enumerate(ks) for s in slots[k]])
        if it in (0, 1, 99):
            apply_checked(st, m, d)
        else:
            st.apply(**d.arrays())
            m.apply(d)
        if it == 1:
            after_second = st.info()["device_bytes"]
    assert st.info()["device_bytes"] <= 2 * after_second, (st.info(), after_second)
    assert st.info()["n_slots"] == 10000
    st.close()


def test_statedb_helper_matches_statedb_root(ctx):
    from phant_b200 import host
    rng = np.random.default_rng(2)
    db = host.StateDB()
    for i in range(200):
        db.db[bytes(rng.integers(0, 256, 20, dtype=np.uint8))] = host.AccountState(
            nonce=i, balance=int(rng.integers(0, 1 << 60)), code=bytes([0x60, i % 256]) * (i % 3),
            storage={int(rng.integers(0, 1 << 60)): int(rng.integers(1, 1 << 60)) for _ in range(i % 30)})
    rs = host.ResidentStateDB(ctx)
    assert rs.load(db) == db.root(ctx)
    addrs = sorted(db.db)
    for blk in range(3):
        touched, changed = {}, {}
        for a in addrs[blk * 20:blk * 20 + 10]:
            s = db.db[a]
            k = next(iter(s.storage), 7)
            changed[a] = {k: 0, 1000 + blk: blk + 1}
            s.storage.pop(k, None)
            s.storage[1000 + blk] = blk + 1
            s.balance += 1
            touched[a] = s
        gone = addrs[150 + blk]
        touched[gone] = None
        del db.db[gone]
        assert rs.apply(touched, changed) == db.root(ctx)
    a = addrs[10]
    db.db[a].storage = {5: 6}
    assert rs.apply({a: db.db[a]}) == db.root(ctx)  # whole storage, replacing what the device held
    rs.close()


def test_premise_round_keeps_the_dense_tops_of_other_accounts(ctx, oracle):
    """One apply where a new account gets a dense top (all buckets built) while another breaks the premise and is rebuilt
    lower: the first account's top must survive for its next incremental apply.  Then a top lowered inside its region
    (L 2 -> 1) must survive a re-layout that another account's new top causes."""
    rng = np.random.default_rng(13)
    st = ctx.resident_state()
    m = StateModel(oracle)
    x, y, z, w = rkey(rng), rkey(rng), rkey(rng), rkey(rng)
    f = (1, u32be(1), ZERO32)
    kx = [rkey(rng) for _ in range(300)]                                          # L 1, random keys
    ky = [bytes([0x30 | int(rng.integers(0, 16))]) + rkey(rng)[1:] for _ in range(300)]  # one first nibble: L 1 breaks
    # w: the second nibble fixed under every first nibble -> L 2 breaks at depth 1, L 1 holds
    kw = [bytes([(int(rng.integers(0, 16)) << 4) | 0x7]) + rkey(rng)[1:] for _ in range(5000)]
    apply_checked(st, m, block(rng, m, {x: f, y: f}, [(x, k, rval(rng)) for k in kx] + [(y, k, rval(rng)) for k in ky]))
    by_bucket = {}
    for k in kx:
        by_bucket.setdefault(k[0] >> 4, k)
    two = list(by_bucket.values())[:2]
    apply_checked(st, m, block(rng, m, {}, [(x, two[0], rval(rng)), (x, two[1], ZERO32)]))
    # w lowered in place; x unchanged beside it
    apply_checked(st, m, block(rng, m, {w: f}, [(w, k, rval(rng)) for k in kw]))
    # z's new top moves every region: x's (L 1) and w's (L 1 inside an L-2 region) are copied
    apply_checked(st, m, block(rng, m, {z: f}, [(z, rkey(rng), rval(rng)) for _ in range(300)]))
    apply_checked(st, m, block(rng, m, {}, [(w, kw[5], rval(rng)), (w, kw[4000], ZERO32), (x, kx[7], rval(rng)), (z, rkey(rng), rval(rng))]))
    st.close()


def test_statedb_helper_recreated_account_in_the_incremental_form(ctx):
    from phant_b200 import host
    db = host.StateDB()
    a, b = b"\x01" * 20, b"\x02" * 20
    db.db[a] = host.AccountState(nonce=1, balance=5, storage={1: 2, 3: 4})
    db.db[b] = host.AccountState(nonce=2, balance=6, storage={5: 6})
    rs = host.ResidentStateDB(ctx)
    assert rs.load(db) == db.root(ctx)
    # a is destroyed and created again in one block: only its new slot is a changed slot
    db.db[a] = host.AccountState(nonce=0, balance=9, storage={7: 8})
    assert rs.apply({a: db.db[a]}, {a: {7: 8}}, recreated={a}) == db.root(ctx)
    with pytest.raises(ValueError):
        rs.apply({a: None}, {}, recreated={a})
    rs.close()
