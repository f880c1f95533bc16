"""Undo on the resident world state (phant_gpu_resident_state_set_journal / _revert) on the GPU: a reverted apply gives back
the root, the counts and the tables the model had before it (tests/resident_state_undo.py states what a record holds)."""
import numpy as np
import pytest

from phant_b200 import gpu
from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel, change_diff, hashed_table, load_diff
from test_gpu_resident_state import apply_checked, block, grow_account, rkey, rval, u32be

pytestmark = pytest.mark.gpu

E_INVALID = -1
EMPTY_ROOT = bytes.fromhex("56e81f171bcc55a6ff8345e692c0f86e5b48e01b996cadc001622fb5e363b421")


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


def counts(m):
    return len(m.acc), sum(len(a.storage) for a in m.acc.values())


def assert_state(st, m, root=None):
    """the device state equals model m: root, and the account and slot counts"""
    want = m.root()
    if root is not None:
        assert root == want
    assert st.root() == want
    info = st.info()
    assert (info["n_accounts"], info["n_slots"]) == counts(m)


def tampered(rng, d):
    """d with one listed balance + 1, or one slot value altered, or (nothing to alter) one more account"""
    up = [i for i, a in enumerate(d.accounts) if not a[1] & DELETE]
    if d.slots and rng.random() < 0.5:
        j = int(rng.integers(0, len(d.slots)))
        ai, sk, v = d.slots[j]
        slots = list(d.slots)
        slots[j] = (ai, sk, u32be(int.from_bytes(v, "big") ^ 0x5a))
        return Diff(d.accounts, slots)
    if up:
        i = up[int(rng.integers(0, len(up)))]
        k, f, n, b, c = d.accounts[i]
        accounts = list(d.accounts)
        accounts[i] = (k, f, n, ((int.from_bytes(b, "big") + 1) % (1 << 256)).to_bytes(32, "big"), c)
        return Diff(accounts, d.slots)
    return Diff(d.accounts + [(rkey(rng), 0, 1, u32be(1), ZERO32)], d.slots)


def test_fixtures_an_invalid_block_is_reverted_then_the_true_one_applied(ctx, oracle, golden):
    g = golden("fixture_states.json.gz")
    rng = np.random.default_rng(31)
    n = 0
    for t in g["tests"]:
        pre, post = hashed_table(oracle.keccak256, g["tables"][t["pre"]]), hashed_table(oracle.keccak256, g["tables"][t["post"]])
        st = ctx.resident_state()
        st.set_journal(1)
        m = StateModel(oracle)
        assert apply_checked(st, m, load_diff(pre)).hex() == t["pre_root"], t["name"]
        d = change_diff(pre, post)
        bad = st.apply(**tampered(rng, d).arrays())
        assert bad.hex() != t["post_root"], t["name"]
        assert st.revert(1).hex() == t["pre_root"], t["name"]
        assert_state(st, m)
        assert st.info()["journal_applies"] == 0
        assert apply_checked(st, m, d).hex() == t["post_root"], t["name"]
        st.close()
        n += 1
    assert n == 84


def test_block_sequence_undone_one_at_a_time_then_a_reorg(ctx, oracle):
    rng = np.random.default_rng(12)
    st = ctx.resident_state()
    st.set_journal(16)
    m = StateModel(oracle)
    keys = [rkey(rng) for _ in range(6000)]
    big, doomed, reborn = keys[0], keys[1], keys[2]
    fields = lambda: (int(rng.integers(0, 1 << 20)), u32be(rng.integers(0, 1 << 60)), rkey(rng))  # noqa: E731
    hist = [(m.copy(), EMPTY_ROOT)]  # (model, root) after each block
    diffs = []

    def step(d):
        diffs.append(d)
        root = apply_checked(st, m, d)
        hist.append((m.copy(), root))

    writes = [(k, rkey(rng), rval(rng)) for k in keys[3:1003] for _ in range(int(rng.integers(1, 10)))]
    writes += grow_account(rng, m, big, 200) + grow_account(rng, m, doomed, 5000) + grow_account(rng, m, reborn, 300)
    step(block(rng, m, {k: fields() for k in keys}, writes))
    for target in (1000, 5000, 70000, 5000, 1000, 200):  # `big`: L 0 -> 1 -> 2 -> 3 and back
        touched = {keys[i]: fields() for i in rng.choice(np.arange(3, 6000), 30, replace=False)}
        w = grow_account(rng, m, big, target)
        small = [keys[i] for i in rng.choice(np.arange(3, 1003), 30, replace=False)]
        w += [(k, list(m.acc[k].storage)[0], rval(rng)) for k in small if m.acc[k].storage]
        w += [(k, rkey(rng), ZERO32) for k in small[:5]]
        step(block(rng, m, touched, w))
    step(block(rng, m, {doomed: (0, ZERO32, ZERO32), reborn: fields()}, [(reborn, rkey(rng), rval(rng)) for _ in range(40)],
               flags={doomed: DELETE, reborn: CLEAR}))
    step(block(rng, m, {}, []))  # an empty block is one apply too
    assert st.info()["journal_applies"] == len(diffs) == 9

    # undo one block at a time, down to the empty state
    for i in range(len(diffs), 0, -1):
        assert st.revert(1) == hist[i - 1][1]
        assert_state(st, hist[i - 1][0])
    assert st.root() == EMPTY_ROOT and st.info()["journal_applies"] == 0
    with pytest.raises(gpu.PhantGpuError) as e:
        st.revert(1)
    assert e.value.code == E_INVALID

    # the same blocks again, then a reorg: undo 4 and apply another 4-block branch on top of the tables the revert left
    for i, d in enumerate(diffs):
        assert st.apply(**d.arrays()) == hist[i + 1][1]
    assert st.revert(4) == hist[len(diffs) - 4][1]
    m = hist[len(diffs) - 4][0].copy()
    assert_state(st, m)
    apply_checked(st, m, block(rng, m, {big: fields()}, grow_account(rng, m, big, 20000)))
    apply_checked(st, m, block(rng, m, {doomed: fields(), reborn: fields()}, [(doomed, rkey(rng), rval(rng)) for _ in range(50)],
                               flags={doomed: CLEAR}))
    apply_checked(st, m, block(rng, m, {reborn: (0, ZERO32, ZERO32)}, [], flags={reborn: DELETE}))
    apply_checked(st, m, block(rng, m, {}, [(big, sk, ZERO32) for sk in list(m.acc[big].storage)[:100]] +
                               [(doomed, sk, rval(rng)) for sk in list(m.acc[doomed].storage)[:100]]))
    assert_state(st, m)
    st.close()


def test_broken_premise_apply_revert_apply(ctx, oracle):
    rng = np.random.default_rng(5)
    st = ctx.resident_state()
    st.set_journal(4)
    m = StateModel(oracle)
    a, b, x = rkey(rng), rkey(rng), rkey(rng)
    f = (1, u32be(1), ZERO32)
    ka = [bytes([0xa0 | int(rng.integers(0, 16))]) + rkey(rng)[1:] for _ in range(300)]  # one first nibble: L 1 breaks
    kb = [b"\x5c" + rkey(rng)[1:] for _ in range(5000)]                                   # one first byte: L 2 lowered twice
    kx = [rkey(rng) for _ in range(300)]
    apply_checked(st, m, block(rng, m, {x: f}, [(x, k, rval(rng)) for k in kx]))
    d = block(rng, m, {a: f, b: f}, [(a, k, rval(rng)) for k in ka] + [(b, k, rval(rng)) for k in kb] + [(x, kx[3], ZERO32)])
    before = m.copy()
    apply_checked(st, m, d)
    assert st.revert(1) == before.root()
    assert_state(st, before)
    m = before
    apply_checked(st, m, d)
    w = [(a, ka[i], rval(rng)) for i in rng.choice(300, 20, replace=False)] + [(b, kb[i], ZERO32) for i in rng.choice(5000, 30, replace=False)]
    d2 = block(rng, m, {}, w + [(x, kx[5], rval(rng))])
    before = m.copy()
    apply_checked(st, m, d2)
    assert st.revert(1) == before.root()
    assert_state(st, before)
    m = before
    apply_checked(st, m, d2)
    st.close()


def test_journal_limits(ctx, oracle):
    rng = np.random.default_rng(6)
    st = ctx.resident_state()
    m = StateModel(oracle)
    f = (1, u32be(3), ZERO32)
    ks = [rkey(rng) for _ in range(8)]
    apply_checked(st, m, Diff([(k, 0) + f for k in ks]))
    with pytest.raises(gpu.PhantGpuError) as e:  # depth 0: nothing to undo
        st.revert(1)
    assert e.value.code == E_INVALID
    assert st.revert(0) == st.root()
    with pytest.raises(gpu.PhantGpuError) as e:
        st.set_journal(1025)
    assert e.value.code == E_INVALID
    st.set_journal(3)
    roots = [st.root()]
    for i in range(5):
        roots.append(apply_checked(st, m, Diff([(ks[i], 0, 10 + i, u32be(i), ZERO32)], [(0, rkey(rng), rval(rng))])))
    assert st.info()["journal_applies"] == 3
    with pytest.raises(gpu.PhantGpuError) as e:
        st.revert(4)
    assert e.value.code == E_INVALID
    assert st.root() == roots[5] and st.info()["journal_applies"] == 3
    assert st.revert(3) == roots[2]
    assert st.revert(0) == roots[2]
    # a refused apply pushes nothing, an empty one pushes a record
    with pytest.raises(gpu.PhantGpuError):
        st.apply(**Diff([(ks[0], 0) + f, (ks[0], 0) + f]).arrays())
    assert st.info()["journal_applies"] == 0
    e0 = np.zeros(0, np.uint8)
    assert st.apply(e0, np.zeros(0, np.uint64), e0, e0) == roots[2]
    assert st.info()["journal_applies"] == 1
    r3 = st.apply(**Diff([(ks[1], 0, 99, u32be(99), ZERO32)]).arrays())
    r4 = st.apply(**Diff([(ks[2], 0, 98, u32be(98), ZERO32)]).arrays())
    assert st.info()["journal_applies"] == 3
    st.set_journal(1)  # keeps only the newest record
    assert st.info()["journal_applies"] == 1
    assert st.revert(1) == r3
    with pytest.raises(gpu.PhantGpuError):
        st.revert(1)
    assert st.root() == r3 != r4
    st.close()


def test_revert_costs_from_the_stats(ctx, oracle):
    rng = np.random.default_rng(22)
    st = ctx.resident_state()
    m = StateModel(oracle)
    big = rkey(rng)
    n = 1_000_000
    sk = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    sv = np.zeros((n, 32), np.uint8)
    sv[:, 31] = 1 + rng.integers(0, 255, n)
    d = Diff([(big, 0, 1, u32be(1), ZERO32)])
    a = d.arrays()
    a.update(slot_account=np.zeros(n, np.uint32), slot_keys32=sk.reshape(-1), slot_vals32=sv.reshape(-1))
    st.apply(**a)
    m.apply(d)
    m.acc[big].storage = {sk[i].tobytes(): sv[i].tobytes() for i in range(n)}
    root0 = st.root()
    assert root0 == m.root()
    st.set_journal(2)
    apply_checked(st, m, Diff([(big, 0, 2, u32be(2), ZERO32)], [(0, sk[5].tobytes(), u32be(99))]))
    ctx.reset_stats()
    assert st.revert(1) == root0
    s = ctx.stats()
    assert s["keccak_msgs"] < 2000, s
    assert s["h2d_bytes"] < 1024, s
    # launches of a revert do not grow with the number of accounts the apply listed
    ks = [rkey(rng) for _ in range(2000)]
    st.apply(**block(rng, m, {k: (1, u32be(1), ZERO32) for k in ks}, [(k, rkey(rng), rval(rng)) for k in ks for _ in range(3)]).arrays())
    launches = []
    for cnt in (10, 2000):
        before = st.root()
        st.apply(**block(rng, m, {k: (2, u32be(cnt), ZERO32) for k in ks[:cnt]}, [(k, rkey(rng), rval(rng)) for k in ks[:cnt]]).arrays())
        ctx.reset_stats()
        assert st.revert(1) == before
        s = ctx.stats()
        assert s["h2d_bytes"] < 1024, s
        launches.append(s["launches"])
    assert launches[1] < 2 * launches[0], launches
    st.close()


def test_device_memory_stays_bounded_over_apply_revert_cycles(ctx, oracle):
    rng = np.random.default_rng(9)
    st = ctx.resident_state()
    m = StateModel(oracle)
    ks = [rkey(rng) for _ in range(5000)]
    slots = {k: [rkey(rng), rkey(rng)] for k in ks}
    apply_checked(st, m, Diff([(k, 0, 0, u32be(1), ZERO32) for k in ks], [(i, s, rval(rng)) for i, k in enumerate(ks) for s in slots[k]]))
    base = st.root()
    st.set_journal(8)
    after_second = None
    for it in range(100):
        d = Diff([(k, 0, it + 1, u32be(int(rng.integers(1, 1 << 62))), ZERO32) for k in ks],
                 [(i, s, rval(rng)) for i, k in enumerate(ks) for s in slots[k]])
        st.apply(**d.arrays())
        assert st.revert(1) == base
        if it == 1:
            after_second = st.info()["device_bytes"]
    info = st.info()
    assert info["device_bytes"] <= 2 * after_second, (info, after_second)
    assert info["journal_applies"] == 0 and info["journal_bytes"] > 0
    assert_state(st, m)
    st.set_journal(0)
    info = st.info()
    assert info["journal_bytes"] == 0 and info["device_bytes"] < after_second
    st.close()
