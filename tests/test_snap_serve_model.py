"""The CPU statement of the snap server's answers (tests/snap_serve_model.py) checked the way a syncing peer checks them, with
the CPU range-proof oracle (tests/range_proof_oracle.py): every account answer, its slim bodies expanded to leaves, is
accepted from its origin with `more` set exactly when accounts follow its last entry; every storage answer's lists are
accepted WHOLE against their storage roots except the one that carries a proof, accepted from its origin.  On the fixture
states and on random states with extensions and embedded leaves."""
import numpy as np

from resident_state_model import Diff, StateModel, hashed_table, load_diff
from snap_serve_model import FF, ZERO, Prover, account_answer, check_account_answer, check_storage_answer, storage_answer

BUDGETS = (0, 1, 36, 37, 100, 500, 4096, 2 << 20)


def add(k, d):
    return ((int.from_bytes(k, "big") + d) % (1 << 256)).to_bytes(32, "big")


def check_state(oracle, m, rng, n_acc=12, n_sto=12):
    kc = oracle.keccak256
    root, pv, keys = m.root(), Prover(oracle, m), sorted(m.acc)
    rich = [k for k in keys if m.acc[k].storage]
    origins = [ZERO] + [add(k, d) for k in (keys if len(keys) <= n_acc else [keys[i] for i in rng.choice(len(keys), n_acc, replace=False)])
                        for d in (-1, 0, 1)]
    for o in origins:
        b = int(rng.choice(BUDGETS))
        accounts, proof = account_answer(m, pv, o, FF, b)
        assert len(accounts) >= 1 or not [k for k in keys if k >= o]
        st, more = check_account_answer(kc, root, o, accounts, proof)
        assert st == 1, (o.hex(), b)
        assert more == bool(accounts and accounts[-1][0] < keys[-1])
    for _ in range(n_sto if rich else 0):
        accts = [rich[i] for i in rng.integers(0, len(rich), int(rng.integers(1, 6)))] + [bytes(rng.integers(0, 256, 32, dtype=np.uint8))]
        sk = sorted(m.acc[accts[0]].storage)
        o = sk[int(rng.integers(0, len(sk)))] if rng.random() < 0.5 else ZERO
        b = int(rng.choice(BUDGETS))
        lists, proof = storage_answer(m, pv, accts, o, FF, b)
        res = check_storage_answer(kc, m, accts, o, lists, proof)
        assert all(s == 1 for s, _ in res), (res, b)


def test_fixture_states(oracle, golden):
    g = golden("fixture_states.json.gz")
    rng = np.random.default_rng(61)
    for name in sorted(g["tables"]):
        m = StateModel(oracle)
        m.apply(load_diff(hashed_table(oracle.keccak256, g["tables"][name])))
        check_state(oracle, m, rng)


def test_random_states(oracle):
    rng = np.random.default_rng(62)
    for t in range(6):
        m = StateModel(oracle)
        d = Diff()
        for i in range(int(rng.integers(1, 300))):
            k = bytearray(rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
            if t % 2:
                k[:30] = b"\x42" * 30  # long shared prefixes: extensions
            d.accounts.append((bytes(k), 0, int(rng.integers(0, 1 << 40)), int(rng.integers(0, 1 << 62)).to_bytes(32, "big"), bytes(32)))
            for _ in range(int(rng.integers(0, 40)) if i % 3 == 0 else 0):
                sk = bytearray(rng.integers(0, 256, 32, dtype=np.uint8).tobytes())
                if t % 2:
                    sk[:31] = b"\x77" * 31  # 1-byte values under a long prefix: embedded leaves
                d.slots.append((len(d.accounts) - 1, bytes(sk), int(rng.integers(1, 200)).to_bytes(32, "big")))
        m.apply(d)
        check_state(oracle, m, rng)
