"""The transition roots at the sizes a client meets: 100k accounts and 1M slots with blocks of 3,000 accounts checked
against the resident world state, 64 blocks in one call, and a 20,000-account state with one 70,000-slot contract checked
against the model and against single-block calls.  The witnesses are cut once per module."""
import numpy as np
import pytest

import oracle_lib
from phant_b200 import gpu
from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel
from transition_oracle import witness

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


def build_state(oracle, rng, n_acc, storage):
    """n_acc accounts; storage = [(account index, slot count)]"""
    m = StateModel(oracle)
    keys = rng.integers(0, 256, (n_acc, 32), dtype=np.uint8)
    d = Diff([(keys[i].tobytes(), 0, i, (i + 1).to_bytes(32, "big"), bytes(32)) for i in range(n_acc)])
    for ai, n in storage:
        sk = rng.integers(0, 256, (n, 32), dtype=np.uint8)
        d.slots += [(ai, sk[j].tobytes(), (j + 1).to_bytes(32, "big")) for j in range(n)]
    m.apply(d)
    return m, d


def block_diff(rng, m, keys, b, n_acc):
    d = Diff()
    for i in rng.choice(len(keys), n_acc, replace=False):
        k = keys[i]
        f = DELETE if i % 50 == 0 else (CLEAR if i % 97 == 0 else 0)
        d.accounts.append((k, f, b + 1000, (b + 7).to_bytes(32, "big"), bytes(32)))
        st = m.acc[k].storage
        if not f & DELETE and st:
            old = sorted(st)
            pick = rng.choice(len(old), min(len(old), 25), replace=False)
            d.slots += [(len(d.accounts) - 1, old[j], (b + 3).to_bytes(32, "big") if n % 5 else ZERO32) for n, j in enumerate(pick)]
            d.slots += [(len(d.accounts) - 1, rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), (b + 9).to_bytes(32, "big"))]
    for _ in range(n_acc // 100):
        d.accounts.append((rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), 0, 1, (1).to_bytes(32, "big"), bytes(32)))
    return d


def one_call(ctx, blocks):
    nodes = list(dict.fromkeys(n for b in blocks for n in b[0]))
    data, off = oracle_lib.csr(nodes, np.uint64)
    d = Diff()
    ablock = []
    for bi, (_, _, bd) in enumerate(blocks):
        base = len(d.accounts)
        d.accounts += bd.accounts
        d.slots += [(base + ai, sk, v) for ai, sk, v in bd.slots]
        ablock += [bi] * len(bd.accounts)
    pre = np.frombuffer(b"".join(b[1] for b in blocks), np.uint8)
    return ctx.transition_roots(data, off, pre, **d.arrays(), account_block=np.array(ablock, np.uint32))


def test_100k_accounts_1m_slots_64_blocks_against_the_resident_world_state(ctx, oracle):
    rng = np.random.default_rng(100)
    # 1M slots: 1,000 contracts of 1,000 slots
    m, full = build_state(oracle, rng, 100_000, [(i * 100, 1000) for i in range(1000)])
    st = ctx.resident_state()
    st.set_journal(1)
    pre = st.apply(**full.arrays())
    assert pre == m.root()
    keys = sorted(m.acc)
    trie = oracle.trie([(k, m.leaf(k)) for k in keys])
    blocks, want = [], []
    for b in range(64):
        d = block_diff(rng, m, keys, b, 3000)
        want.append(st.apply(**d.arrays()))
        st.revert(1)
        blocks.append((witness(oracle, m, d, account_trie=trie), pre, d))
    st.close()
    ctx.reset_stats()
    roots, status = one_call(ctx, blocks[:1])
    one = ctx.stats()["launches"]
    assert status[0] == 1 and roots[0].tobytes() == want[0]
    ctx.reset_stats()
    roots, status = one_call(ctx, blocks)
    many = ctx.stats()["launches"]
    assert list(status) == [1] * 64
    assert [r.tobytes() for r in roots] == want
    assert many < 2 * one, (many, one)


def test_20k_accounts_with_a_70k_slot_contract_against_the_model(ctx, oracle):
    rng = np.random.default_rng(20)
    m, _ = build_state(oracle, rng, 20_000, [(7, 70_000)] + [(i, 50) for i in range(100, 20_000, 400)])
    pre = m.root()
    keys = sorted(m.acc)
    trie = oracle.trie([(k, m.leaf(k)) for k in keys])
    big = next(k for k in keys if len(m.acc[k].storage) == 70_000)
    blocks, want = [], []
    for b in range(6):
        d = block_diff(rng, m, keys, b, 1500)
        ai = next((i for i, a in enumerate(d.accounts) if a[0] == big), None)
        if ai is None:
            d.accounts.append((big, 0, 5, (5).to_bytes(32, "big"), bytes(32)))
            ai = len(d.accounts) - 1
        if not d.accounts[ai][1] & DELETE:
            old = sorted(m.acc[big].storage)
            d.slots = [s for s in d.slots if s[0] != ai]
            d.slots += [(ai, old[j], ZERO32 if j % 3 == 0 else (b + 11).to_bytes(32, "big")) for j in rng.choice(70_000, 3000, replace=False)]
            d.slots += [(ai, rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), (1).to_bytes(32, "big")) for _ in range(1000)]
        mm = m.copy()
        mm.apply(d)
        want.append(mm.root())
        blocks.append((witness(oracle, m, d, account_trie=trie), pre, d))
    roots, status = one_call(ctx, blocks)
    assert list(status) == [1] * 6 and [r.tobytes() for r in roots] == want
    for bi, b in enumerate(blocks):
        r1, s1 = one_call(ctx, [b])
        assert s1[0] == 1 and r1[0].tobytes() == want[bi], bi
