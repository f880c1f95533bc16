"""The transition roots (phant_gpu_transition_roots) on the GPU against the CPU statement (tests/transition_oracle.py), the
world-state model and the fixture headers: one call validates many independent blocks, each against its own parent root."""

import numpy as np
import pytest

import oracle_lib
from phant_b200 import gpu
from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel, change_diff, hashed_table, load_diff
from test_transition_model import collapse_cases, random_case
from transition_oracle import transition, witness

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


def call(ctx, blocks, extra_nodes=()):
    """blocks: [(node list, pre_root, Diff)] -> (roots, status, storage roots) of ONE call over the union of the node sets"""
    nodes = list(dict.fromkeys([n for b in blocks for n in b[0]] + list(extra_nodes)))
    data, off = oracle_lib.csr(nodes, np.uint64)
    d = Diff()
    ablock = []
    for bi, (_, _, bd) in enumerate(blocks):
        base = len(d.accounts)
        d.accounts += bd.accounts
        d.slots += [(base + ai, sk, v) for ai, sk, v in bd.slots]
        ablock += [bi] * len(bd.accounts)
    pre = np.frombuffer(b"".join(b[1] for b in blocks), np.uint8)
    return ctx.transition_roots(data, off, pre, **d.arrays(), account_block=np.array(ablock, np.uint32), storage_roots=True)


def check_blocks(ctx, oracle, blocks):
    """one call over all blocks; each block's result is the CPU statement's over the union of the node sets"""
    roots, status, sroots = call(ctx, blocks)
    union = list(dict.fromkeys(n for b in blocks for n in b[0]))
    k = 0
    for bi, (_, pre, d) in enumerate(blocks):
        st, root, want_sroots, _ = transition(oracle, union, pre, d)
        assert status[bi] == st, bi
        assert roots[bi].tobytes() == (root if st == 1 else ZERO32), bi
        for i in range(len(d.accounts)):
            assert sroots[k + i].tobytes() == (want_sroots[i] if st == 1 else ZERO32), (bi, i)
        k += len(d.accounts)
    return roots, status


def test_all_fixtures_in_one_call(ctx, oracle, golden):
    g = golden("fixture_states.json.gz")
    blocks, models = [], []
    for t in g["tests"]:
        pre, post = hashed_table(oracle.keccak256, g["tables"][t["pre"]]), hashed_table(oracle.keccak256, g["tables"][t["post"]])
        m = StateModel(oracle)
        m.apply(load_diff(pre))
        d = change_diff(pre, post)
        blocks.append((witness(oracle, m, d), bytes.fromhex(t["pre_root"]), d))
        m.apply(d)
        models.append(m)
    assert len(blocks) == 84
    roots, status, sroots = call(ctx, blocks)
    k = 0
    for bi, t in enumerate(g["tests"]):
        assert status[bi] == 1 and roots[bi].tobytes().hex() == t["post_root"], t["name"]
        for a in blocks[bi][2].accounts:
            assert sroots[k].tobytes() == (ZERO32 if a[1] & DELETE else models[bi].storage_root(a[0])), t["name"]
            k += 1


def test_random_blocks_match_the_model_and_single_block_calls(ctx, oracle):
    rng = np.random.default_rng(3)
    blocks, want = [], []
    for _ in range(6):
        m, d = random_case(oracle, rng, n_acc=300, n_slots=60)
        blocks.append((witness(oracle, m, d), m.root(), d))
        m.apply(d)
        want.append(m.root())
    # an incomplete witness (status 3: a state of its own, with a node the computation reads dropped) and a pre-root over a
    # node that breaks R2 (status 0) in the same batch
    m, d = random_case(oracle, rng, n_acc=300, n_slots=60)
    nodes = witness(oracle, m, d)
    _, _, _, reads = transition(oracle, nodes, m.root(), d)
    drop = next(i for i, n in enumerate(nodes) if oracle.keccak256(n) in reads)
    blocks.append((nodes[:drop] + nodes[drop + 1:], m.root(), d))
    bad = b"\xc3\x80\x80"
    blocks.append(([bad], oracle.keccak256(bad), d))
    roots, status = check_blocks(ctx, oracle, blocks)
    assert list(status[:6]) == [1] * 6 and [roots[i].tobytes() for i in range(6)] == want
    assert status[6] == 3 and status[7] == 0
    for bi, b in enumerate(blocks):
        r1, s1, _ = call(ctx, [b])
        assert s1[0] == status[bi] and r1[0].tobytes() == roots[bi].tobytes(), bi


def test_dropping_any_node_never_gives_a_wrong_root(ctx, oracle):
    rng = np.random.default_rng(8)
    m, d = random_case(oracle, rng, n_acc=24, n_slots=12)
    pre = m.root()
    nodes = witness(oracle, m, d)
    m.apply(d)
    blocks = [(nodes[:i] + nodes[i + 1:], pre, d) for i in range(len(nodes))] + [(nodes, pre, d)]
    roots, status, _ = call(ctx, blocks[-1:])
    assert status[0] == 1 and roots[0].tobytes() == m.root()
    for b in blocks[:-1]:  # one call per dropped node: the blocks of one call share their nodes
        r, s, _ = call(ctx, [b])
        st, root, _, _ = transition(oracle, *b)
        assert s[0] == st and s[0] in (1, 3)
        assert r[0].tobytes() == (m.root() if s[0] == 1 else ZERO32)


def crafted_state(oracle, keys, slots=()):
    m = StateModel(oracle)
    d = Diff([(k, 0, 1, (1).to_bytes(32, "big"), bytes(32)) for k in keys])
    d.slots = list(slots)
    m.apply(d)
    return m


def test_crafted_structures(ctx, oracle):
    rng = np.random.default_rng(21)
    rk = lambda: bytes(rng.integers(0, 256, 32, dtype=np.uint8))  # noqa: E731
    pair = rk()
    pairs = [pair[:31] + bytes([(pair[31] & 0xF0) | v]) for v in (1, 2, 3)]  # differ only in the last nibble
    prefix = rk()[:5]
    under = [prefix + rk()[5:] for _ in range(700)]  # 700 keys under one 5-byte prefix
    base = [rk() for _ in range(40)]
    m = crafted_state(oracle, base + pairs + under)
    cases = [
        Diff([(pairs[0], DELETE, 0, ZERO32, ZERO32)]),                                    # a last-nibble branch keeps two children
        Diff([(pairs[0], DELETE, 0, ZERO32, ZERO32), (pairs[1], DELETE, 0, ZERO32, ZERO32)]),  # it collapses onto a leaf
        Diff([(k, DELETE, 0, ZERO32, ZERO32) for k in under[:699]]),                      # down to one key under the prefix
        Diff([(prefix + rk()[5:], 0, 5, (5).to_bytes(32, "big"), bytes(32)) for _ in range(50)]),  # inserts under the prefix
        Diff([(k, DELETE, 0, ZERO32, ZERO32) for k in base + pairs + under]),              # down to empty
        Diff([(k, DELETE, 0, ZERO32, ZERO32) for k in base + pairs + under[1:]]),          # down to a single leaf
        Diff([(pair[:31] + bytes([(pair[31] & 0xF0) | 9]), 0, 2, (2).to_bytes(32, "big"), bytes(32))]),  # last-nibble insert
    ]
    blocks = [(witness(oracle, m, d), m.root(), d) for d in cases]
    roots, status = check_blocks(ctx, oracle, blocks)
    for bi, (_, _, d) in enumerate(blocks):
        mm = m.copy()
        mm.apply(d)
        assert status[bi] == 1 and roots[bi].tobytes() == mm.root(), bi


def test_collapse_onto_each_kind_of_node(ctx, oracle):
    """a deleted key's only surviving sibling is a hashed extension, a hashed branch, an extension over an embedded branch, or
    an embedded leaf: each against the model, then with every witness node dropped in turn against the CPU statement"""
    for name, m, d, kind in collapse_cases(oracle):
        nodes = witness(oracle, m, d)
        seen = []
        transition(oracle, nodes, m.root(), d, collapses=seen)
        assert (kind in seen) if kind else not seen, name
        want = m.copy()
        want.apply(d)
        roots, status = check_blocks(ctx, oracle, [(nodes, m.root(), d)])
        assert status[0] == 1 and roots[0].tobytes() == want.root(), name
        for i in range(len(nodes)):
            b = (nodes[:i] + nodes[i + 1:], m.root(), d)
            r, s, _ = call(ctx, [b])
            st, root, _, _ = transition(oracle, *b)
            assert s[0] == st and s[0] in (1, 3), (name, i)
            assert r[0].tobytes() == (want.root() if st == 1 else ZERO32), (name, i)


def test_extension_split_without_the_node_below(ctx, oracle):
    """two keys sharing 10 nibbles sit under an extension; an insert that splits it needs only the extension"""
    a = bytes.fromhex("abcdef0123") + bytes(range(27))
    b = a[:5] + bytes([0x44]) + a[6:]
    m = crafted_state(oracle, [a, b] + [bytes([i * 16]) + bytes(31) for i in range(1, 4)])
    new = a[:3] + bytes([0xe0]) + a[4:]
    d = Diff([(new, 0, 1, (1).to_bytes(32, "big"), bytes(32))])
    nodes = witness(oracle, m, d)
    trie = oracle.trie([(k, m.leaf(k)) for k in sorted(m.acc)])
    below = set(trie.prove(a)) - set(nodes)
    assert below  # the branch below the extension is not in the witness
    roots, status = check_blocks(ctx, oracle, [(nodes, m.root(), d)])
    m.apply(d)
    assert status[0] == 1 and roots[0].tobytes() == m.root()


def test_malformed_nodes_and_junk(ctx, oracle):
    rng = np.random.default_rng(4)
    m, d = random_case(oracle, rng, n_acc=40, n_slots=10)
    nodes = witness(oracle, m, d)
    junk = [bytes(rng.integers(0, 256, int(rng.integers(1, 200)), dtype=np.uint8)) for _ in range(50)]
    r0, s0, _ = call(ctx, [(nodes, m.root(), d)])
    r1, s1, _ = call(ctx, [(nodes, m.root(), d)], extra_nodes=junk)
    assert s0[0] == s1[0] == 1 and r0[0].tobytes() == r1[0].tobytes()
    # R3: a branch child that is neither empty, a hash nor embedded; an account body that is not a 4-item list
    br = b"\xd1" + b"\x81\x01" + b"\x80" * 15
    leaf = gpu_leaf(bytes(32), b"\x82\x01\x02")
    blocks = [([br], oracle.keccak256(br), Diff([(bytes(32), 0, 1, ZERO32, ZERO32)])),
              ([leaf], oracle.keccak256(leaf), Diff([(bytes(32), 0, 1, ZERO32, ZERO32)]))]
    _, status = check_blocks(ctx, oracle, blocks)
    assert list(status) == [0, 0]


def gpu_leaf(key, value):
    from helpers import _hp, rlp_list, rlp_str
    from transition_oracle import nibbles
    return rlp_list([rlp_str(_hp(nibbles(key), True)), rlp_str(value)])


def test_refusals_write_nothing(ctx, oracle):
    k = bytes(range(32))
    good = Diff([(k, 0, 1, ZERO32, ZERO32)])
    data, off = oracle_lib.csr([b"\xc0"], np.uint64)
    pre = np.frombuffer(oracle.keccak256(b"\xc0"), np.uint8).copy()

    def run(d, ablock=None, nb=1):
        a = d.arrays()
        keep = [a]  # noqa: F841 -- the arrays must outlive the call
        t = gpu.Transition(1, data.ctypes.data, off.ctypes.data, int(off[-1]), nb, pre.ctypes.data,
                           None if ablock is None else ablock.ctypes.data)
        sd = gpu.StateDiff(len(d.accounts), *[a[f] if a[f] is None else a[f].ctypes.data for f in
                                              ("account_keys32", "account_flags", "nonce", "balance32", "code_hash32")],
                           len(d.slots), *[None if a[f] is None else a[f].ctypes.data for f in ("slot_account", "slot_keys32", "slot_vals32")])
        roots = np.full((max(nb, 1), 32), 0xAB, np.uint8)
        status = np.full(max(nb, 1), 0xAB, np.uint8)
        sroots = np.full((max(len(d.accounts), 1), 32), 0xAB, np.uint8)
        rc = ctx.transition_roots_raw(t, sd, roots, status, sroots)
        return rc, roots, status, sroots

    rc, roots, status, _ = run(good)
    assert rc == 0 and status[0] in (0, 1, 3)
    bad = [
        (Diff([(k, 0, 1, ZERO32, ZERO32), (k, 0, 2, ZERO32, ZERO32)]), None, 1),              # an account twice in one block
        (Diff([(k, 0, 1, ZERO32, ZERO32)], [(0, k, ZERO32), (0, k, ZERO32)]), None, 1),       # a slot twice
        (Diff([(k, 0, 1, ZERO32, ZERO32)], [(1, k, ZERO32)]), None, 1),                       # slot_account out of range
        (Diff([(k, DELETE, 0, ZERO32, ZERO32)], [(0, k, ZERO32)]), None, 1),                  # a slot of a DELETE account
        (Diff([(k, 8, 1, ZERO32, ZERO32)]), None, 1),                                         # unknown flag bits
        (good, np.array([1], np.uint32), 1),                                                  # account_block >= n_blocks
        (good, None, 0),                                                                      # no blocks
    ]
    for i, (d, ab, nb) in enumerate(bad):
        rc, roots, status, sroots = run(d, ab, nb)
        assert rc == -1, i
        assert (roots == 0xAB).all() and (status == 0xAB).all() and (sroots == 0xAB).all(), i
    # device pointers: the diff's keys, or the node set, in GPU memory
    torch = pytest.importorskip("torch")
    a = good.arrays()
    dev_keys = torch.from_numpy(a["account_keys32"].copy()).cuda()
    dev_nodes = torch.from_numpy(data.copy()).cuda()
    t = gpu.Transition(1, data.ctypes.data, off.ctypes.data, int(off[-1]), 1, pre.ctypes.data, None)
    for keys_ptr, nodes_ptr in ((dev_keys.data_ptr(), data.ctypes.data), (a["account_keys32"].ctypes.data, dev_nodes.data_ptr())):
        t.nodes = nodes_ptr
        sd = gpu.StateDiff(1, keys_ptr, None, a["nonce"].ctypes.data, a["balance32"].ctypes.data, a["code_hash32"].ctypes.data, 0, None,
                           None, None)
        roots = np.full((1, 32), 0xAB, np.uint8)
        status = np.full(1, 0xAB, np.uint8)
        assert ctx.transition_roots_raw(t, sd, roots, status) == -1
        assert (roots == 0xAB).all() and (status == 0xAB).all()
    # the same account in two blocks is fine
    rc, _, status, _ = run(Diff([(k, 0, 1, ZERO32, ZERO32), (k, 0, 2, ZERO32, ZERO32)]), np.array([0, 1], np.uint32), 2)
    assert rc == 0


def test_against_the_resident_world_state(ctx, oracle):
    """blocks applied to the resident world state, reverted in between, give the roots T computes from witnesses"""
    rng = np.random.default_rng(9)
    m, _ = random_case(oracle, rng, n_acc=2000, n_slots=200)
    st = ctx.resident_state()
    st.set_journal(1)
    full = load_diff({k: (a.nonce, a.balance, a.code_hash, dict(a.storage)) for k, a in m.acc.items()})
    pre = st.apply(**full.arrays())
    assert pre == m.root()
    blocks, want = [], []
    keys = sorted(m.acc)
    for b in range(8):
        d = Diff()
        for i in rng.choice(len(keys), 150, replace=False):
            k = keys[i]
            f = DELETE if i % 9 == 0 else (CLEAR if i % 11 == 0 else 0)
            d.accounts.append((k, f, b, (b + 1).to_bytes(32, "big"), bytes(32)))
            if not f & DELETE and m.acc[k].storage:
                old = sorted(m.acc[k].storage)
                d.slots += [(len(d.accounts) - 1, sk, (b + 7).to_bytes(32, "big")) for sk in old[:3]]
                d.slots += [(len(d.accounts) - 1, sk, ZERO32) for sk in old[3:5]]
        want.append(st.apply(**d.arrays()))
        st.revert(1)
        blocks.append((witness(oracle, m, d), pre, d))
    ctx.reset_stats()
    roots, status, _ = call(ctx, blocks)
    launches_many = ctx.stats()["launches"]
    assert list(status) == [1] * 8 and [r.tobytes() for r in roots] == want
    ctx.reset_stats()
    call(ctx, blocks[:1])
    assert launches_many < 2 * ctx.stats()["launches"]
    st.close()


def test_host_transition_root(ctx, oracle):
    """host.transition_root on a witness blob: the witness of a two-account state, one account changed and one created"""
    from phant_b200 import host
    a1, a2, a3 = bytes(range(20)), bytes(range(1, 21)), bytes(range(2, 22))
    m = StateModel(oracle)
    empty_code = oracle.keccak256(b"")
    m.apply(Diff([(oracle.keccak256(a), 0, 1, (5).to_bytes(32, "big"), empty_code) for a in (a1, a2)]))
    d = Diff([(oracle.keccak256(a1), 0, 2, (9).to_bytes(32, "big"), empty_code), (oracle.keccak256(a3), 0, 0, (1).to_bytes(32, "big"), empty_code)])
    blob = host.encode_witness([], [], witness(oracle, m, d))
    parent = m.root()
    root, status = host.transition_root(ctx, parent, blob, {a1: host.AccountState(2, 9, b""), a3: host.AccountState(0, 1, b"")})
    m.apply(d)
    assert status == 1 and root == m.root()
