"""The Python world-state model the resident-state GPU tests compare against, pinned to the fixtures and to the oracle's S."""
import numpy as np

from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel, change_diff, hashed_table, load_diff


def test_model_reproduces_every_fixture_root(oracle, golden):
    g = golden("fixture_states.json.gz")
    n = 0
    for t in g["tests"]:
        pre, post = hashed_table(oracle.keccak256, g["tables"][t["pre"]]), hashed_table(oracle.keccak256, g["tables"][t["post"]])
        m = StateModel(oracle)
        m.apply(load_diff(pre))
        assert m.root().hex() == t["pre_root"], t["name"]
        m.apply(change_diff(pre, post))
        assert m.root().hex() == t["post_root"], t["name"]
        fresh = StateModel(oracle)
        fresh.apply(load_diff(post))
        assert fresh.root() == m.root()
        n += 1
    assert n == 84


def random_table(rng, n):
    out = []
    for _ in range(n):
        st = {}
        for _ in range(int(rng.integers(0, 40))):
            v = bytes(rng.integers(0, 256, int(rng.integers(1, 33)), dtype=np.uint8)).rjust(32, b"\x00")
            st[bytes(rng.integers(0, 256, 32, dtype=np.uint8)).hex()] = v.hex()
        out.append(dict(address=bytes(rng.integers(0, 256, 20, dtype=np.uint8)).hex(), nonce=int(rng.integers(0, 1 << 40)),
                        balance=bytes(rng.integers(0, 256, 32, dtype=np.uint8)).rjust(32, b"\x00").hex(),
                        code=bytes(rng.integers(0, 256, int(rng.integers(0, 50)), dtype=np.uint8)).hex(), storage=st))
    return out


def test_model_equals_oracle_state_root_on_random_tables(oracle):
    rng = np.random.default_rng(5)
    for n in (1, 2, 7, 60, 300):
        tab = random_table(rng, n)
        m = StateModel(oracle)
        m.apply(load_diff(hashed_table(oracle.keccak256, tab)))
        assert m.root() == oracle.state_root(tab), n


def test_model_semantics_of_flags_and_zero_values(oracle):
    k = [bytes([i]) * 32 for i in range(1, 4)]
    s = [bytes([0x10 + i]) * 32 for i in range(4)]
    one = (1).to_bytes(32, "big")
    m = StateModel(oracle)
    m.apply(Diff([(k[0], 0, 1, one, ZERO32), (k[1], 0, 2, one, ZERO32)], [(0, s[0], one), (0, s[1], one), (1, s[2], ZERO32)]))
    assert len(m.acc[k[0]].storage) == 2 and m.acc[k[1]].storage == {}
    m.apply(Diff([(k[0], CLEAR, 1, one, ZERO32)], [(0, s[3], one)]))
    assert list(m.acc[k[0]].storage) == [s[3]]
    m.apply(Diff([(k[0], DELETE, 0, ZERO32, ZERO32), (k[2], DELETE, 0, ZERO32, ZERO32)]))
    assert list(m.acc) == [k[1]]
