"""The undo statement (tests/resident_state_undo.py) on the CPU: applying a diff and then its inverse gives back the model
exactly, on every fixture and on random block sequences undone newest first."""
import numpy as np

from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel, change_diff, hashed_table, load_diff
from resident_state_undo import inverse, snapshot


def test_inverse_takes_every_fixture_back_to_pre(oracle, golden):
    g = golden("fixture_states.json.gz")
    n = 0
    for t in g["tests"]:
        pre, post = hashed_table(oracle.keccak256, g["tables"][t["pre"]]), hashed_table(oracle.keccak256, g["tables"][t["post"]])
        m = StateModel(oracle)
        m.apply(load_diff(pre))
        loaded = snapshot(m)
        d = change_diff(pre, post)
        inv = inverse(m, d)
        m.apply(d)
        assert m.root().hex() == t["post_root"], t["name"]
        m.apply(inv)
        assert m.root().hex() == t["pre_root"], t["name"]
        assert snapshot(m) == loaded, t["name"]
        n += 1
    assert n == 84


def _val(rng):
    return bytes(rng.integers(0, 256, int(rng.integers(1, 33)), dtype=np.uint8)).rjust(32, b"\x00").replace(ZERO32, b"\x00" * 31 + b"\x01")


def _random_diff(rng, m, keys):
    """every kind of listing: upserts of present and absent accounts, DELETE of present and absent ones, CLEAR_STORAGE
    (destroyed and re-created in one diff), slot writes, deletes of present slots and zero writes to absent ones"""
    picked = rng.choice(len(keys), int(rng.integers(1, 12)), replace=False)
    accounts, slots = [], []
    for i in picked:
        k = keys[i]
        r = rng.random()
        flags = DELETE if r < 0.15 else CLEAR if r < 0.3 else 0
        accounts.append((k, flags, int(rng.integers(0, 1 << 40)), _val(rng), bytes(rng.integers(0, 256, 32, dtype=np.uint8))))
        if flags & DELETE:
            continue
        j = len(accounts) - 1
        have = list(m.acc[k].storage) if k in m.acc else []
        chosen = {}
        for _ in range(int(rng.integers(0, 8))):
            c = rng.random()
            if have and c < 0.4:
                chosen[have[int(rng.integers(0, len(have)))]] = ZERO32 if rng.random() < 0.5 else _val(rng)
            elif c < 0.6:
                chosen[bytes(rng.integers(0, 256, 32, dtype=np.uint8))] = ZERO32  # a zero write to an absent slot
            else:
                chosen[bytes(rng.integers(0, 256, 32, dtype=np.uint8))] = _val(rng)
        slots += [(j, sk, v) for sk, v in chosen.items()]
    return Diff(accounts, slots)


def test_random_sequences_undone_newest_first(oracle):
    rng = np.random.default_rng(17)
    for _ in range(4):
        keys = [bytes(rng.integers(0, 256, 32, dtype=np.uint8)) for _ in range(16)]
        m = StateModel(oracle)
        history = []
        for _ in range(25):
            d = _random_diff(rng, m, keys)
            history.append((snapshot(m), m.root(), inverse(m, d)))
            m.apply(d)
        while history:
            before, root, inv = history.pop()
            assert not any(inv.accounts[ai][1] & DELETE for ai, _, _ in inv.slots)
            assert len({(ai, sk) for ai, sk, _ in inv.slots}) == len(inv.slots)
            m.apply(inv)
            assert snapshot(m) == before
            assert m.root() == root


def test_inverse_of_each_listing_kind(oracle):
    one, two = (1).to_bytes(32, "big"), (2).to_bytes(32, "big")
    k = [bytes([i]) * 32 for i in range(1, 6)]
    s = [bytes([0x10 + i]) * 32 for i in range(4)]
    m = StateModel(oracle)
    m.apply(Diff([(k[0], 0, 1, one, ZERO32), (k[1], 0, 2, one, ZERO32), (k[2], 0, 3, one, ZERO32)],
                 [(0, s[0], one), (0, s[1], one), (1, s[2], one), (2, s[3], two)]))
    d = Diff([(k[0], 0, 9, two, ZERO32), (k[1], DELETE, 0, ZERO32, ZERO32), (k[2], CLEAR, 4, two, ZERO32), (k[3], 0, 1, one, ZERO32),
              (k[4], DELETE, 0, ZERO32, ZERO32)],
             [(0, s[0], ZERO32), (0, s[2], two), (2, s[0], one), (3, s[1], one)])
    inv = inverse(m, d)
    assert inv.accounts == [(k[0], 0, 1, one, ZERO32), (k[1], CLEAR, 2, one, ZERO32), (k[2], CLEAR, 3, one, ZERO32),
                            (k[3], DELETE, 0, ZERO32, ZERO32)]
    assert sorted(inv.slots) == sorted([(0, s[0], one), (0, s[2], ZERO32), (1, s[2], one), (2, s[3], two)])
