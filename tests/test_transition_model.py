"""The CPU statement of the transition roots (tests/transition_oracle.py) pinned to the fixture headers and to the world-state
model: on a sufficient witness its root is the model's root after the diff; with one node dropped it gives status 3 exactly
when the full computation read that node, and the same root otherwise."""
import numpy as np

from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel, change_diff, hashed_table, load_diff
from transition_oracle import transition, witness


def model_of(oracle, h):
    m = StateModel(oracle)
    m.apply(load_diff(h))
    return m


def test_fixtures_give_the_header_post_root(oracle, golden):
    g = golden("fixture_states.json.gz")
    n = 0
    for t in g["tests"]:
        pre, post = hashed_table(oracle.keccak256, g["tables"][t["pre"]]), hashed_table(oracle.keccak256, g["tables"][t["post"]])
        m = model_of(oracle, pre)
        d = change_diff(pre, post)
        st, root, sroots, _ = transition(oracle, witness(oracle, m, d), bytes.fromhex(t["pre_root"]), d)
        m.apply(d)
        assert st == 1 and root.hex() == t["post_root"] == m.root().hex(), t["name"]
        for i, a in enumerate(d.accounts):
            assert sroots[i] == (ZERO32 if a[1] & DELETE else m.storage_root(a[0])), (t["name"], i)
        n += 1
    assert n == 84


def random_case(oracle, rng, n_acc=60, n_slots=40):
    m = StateModel(oracle)
    d0 = Diff()
    keys = [bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(n_acc)]
    for i, k in enumerate(keys):
        d0.accounts.append((k, 0, i, (i + 1).to_bytes(32, "big"), bytes(32)))
        if i % 7 == 0:
            d0.slots += [(i, bytes(rng.integers(0, 256, 32, dtype=np.uint8)), (j + 1).to_bytes(32, "big")) for j in range(n_slots)]
    m.apply(d0)
    d = Diff()
    for i, k in enumerate(keys[:20]):
        f = DELETE if i % 5 == 1 else (CLEAR if i % 7 == 3 else 0)
        d.accounts.append((k, f, 99, (7).to_bytes(32, "big"), bytes(32)))
        a = m.acc[k]
        if not f & DELETE:
            old = sorted(a.storage)
            d.slots += [(len(d.accounts) - 1, sk, ZERO32) for sk in old[: len(old) // 2]]
            d.slots += [(len(d.accounts) - 1, bytes(rng.integers(0, 256, 32, dtype=np.uint8)), (5).to_bytes(32, "big")) for _ in range(3)]
    for _ in range(5):
        d.accounts.append((bytes(rng.integers(0, 256, 32, dtype=np.uint8)), 0, 1, (1).to_bytes(32, "big"), bytes(32)))
    return m, d


def test_random_states_give_the_model_root(oracle):
    rng = np.random.default_rng(11)
    for _ in range(4):
        m, d = random_case(oracle, rng)
        pre = m.root()
        st, root, _, _ = transition(oracle, witness(oracle, m, d), pre, d)
        m.apply(d)
        assert st == 1 and root == m.root()


def test_dropping_a_node_gives_status_3_exactly_when_it_was_read(oracle):
    rng = np.random.default_rng(5)
    m, d = random_case(oracle, rng, n_acc=24, n_slots=12)
    pre = m.root()
    nodes = witness(oracle, m, d)
    st, root, _, reads = transition(oracle, nodes, pre, d)
    assert st == 1
    for i, nd in enumerate(nodes):
        st2, root2, _, _ = transition(oracle, nodes[:i] + nodes[i + 1:], pre, d)
        if oracle.keccak256(nd) in reads:
            assert st2 == 3 and root2 is None, i
        else:
            assert st2 == 1 and root2 == root, i


def collapse_cases(oracle):
    """crafted states in which deleting one key leaves its branch with one child, and the diff that does it:
    [(name, model, diff, the kind of node the surviving child must collapse as, or None when it is embedded)]"""
    rng = np.random.default_rng(31)
    rk = lambda n=32: bytes(rng.integers(0, 256, n, dtype=np.uint8))  # noqa: E731
    one = (1).to_bytes(32, "big")
    base = [bytes([v << 4]) + rk(31) for v in range(1, 6)]  # the root is a branch
    x = b"\xab" + rk(31)                                   # the key that goes; its sibling sits under nibbles "ac"

    def state(acc_keys, slots=()):
        m = StateModel(oracle)
        d = Diff([(k, 0, 1, one, bytes(32)) for k in acc_keys])
        d.slots = list(slots)
        m.apply(d)
        return m

    out = []
    ext = [b"\xac\x12\x34\x56" + bytes([v]) + rk(27) for v in (0x10, 0x20)]  # "ac123456", then a branch: a hashed extension
    m = state(base + [x] + ext)
    out.append(("hashed extension", m, Diff([(x, DELETE, 0, ZERO32, ZERO32)]), "ext"))
    br = [b"\xac" + bytes([v]) + rk(30) for v in (0x10, 0x20)]  # "ac" is itself a branch, referenced by hash
    m = state(base + [x] + br)
    out.append(("hashed branch", m, Diff([(x, DELETE, 0, ZERO32, ZERO32)]), "branch"))
    # storage: "ac" + 61 shared nibbles, then two leaves of one-byte values -- a branch small enough to be embedded in the
    # extension above it
    owner = base[0]
    tail = rk(30)
    emb = [b"\xac" + tail + bytes([0x50 | v]) for v in (1, 2)]
    sx = b"\xab" + rk(31)
    m = state(base, [(0, k, one) for k in [sx] + emb + [rk() for _ in range(4)]])
    out.append(("extension over an embedded branch", m, Diff([(owner, 0, 1, one, bytes(32))], [(0, sx, ZERO32)]), "ext"))
    # storage: three keys that differ only in the last nibble; two go and the branch collapses onto the embedded third
    emb3 = [b"\xac" + tail + bytes([0x50 | v]) for v in (1, 2, 3)]
    m = state(base, [(0, k, one) for k in emb3 + [rk() for _ in range(4)]])
    out.append(("embedded leaf", m, Diff([(owner, 0, 1, one, bytes(32))], [(0, emb3[0], ZERO32), (0, emb3[1], ZERO32)]), None))
    return out


def test_collapse_onto_each_kind_of_node(oracle):
    for name, m, d, kind in collapse_cases(oracle):
        nodes = witness(oracle, m, d)
        seen = []
        st, root, _, reads = transition(oracle, nodes, m.root(), d, collapses=seen)
        want = m.copy()
        want.apply(d)
        assert st == 1 and root == want.root(), name
        assert (kind in seen) if kind else not seen, (name, seen)
        for i, nd in enumerate(nodes):
            st2, root2, _, _ = transition(oracle, nodes[:i] + nodes[i + 1:], m.root(), d)
            assert (st2, root2) == ((3, None) if oracle.keccak256(nd) in reads else (1, root)), (name, i)
