"""The CPU statement of the range-proof check (tests/range_proof_oracle.py) pinned to the truth on tries whose contents are
known: every answer served honestly is accepted with the right `more`, and no mutation of one is accepted unless it is still
exactly the trie's contents in its range."""
import numpy as np
import pytest

from range_proof_corpus import (FF32, KnownTrie, accept_cases, awkward_tries, fixture_tries, key_after, mutation_cases, random_tries,
                                truth)
from range_proof_oracle import verify_range


def check_accepts(oracle, t, limit=None, rng=None):
    n = 0
    for origin, ents, nodes, whole, more in accept_cases(t, limit=limit, rng=rng):
        assert truth(t, origin, ents, whole) == (True, more)
        got = verify_range(oracle.keccak256, nodes, t.root, origin, ents, whole)
        assert got == (1, more), (t.name, origin.hex(), len(ents), whole, got)
        n += 1
    return n


def check_mutations(oracle, t, rng):
    names = set()
    for name, root, origin, ents, nodes, whole in mutation_cases(t, rng):
        st, more = verify_range(oracle.keccak256, nodes, root, origin, ents, whole)
        assert st in (0, 1, 3)
        true, want_more = truth(t, origin, ents, whole) if root == t.root else (False, False)
        if name == "drop-last" and true:
            assert st != 1 or more == want_more == 1, (t.name, name)
        else:
            assert st != 1, (t.name, name, origin.hex())
        names.add(name.rstrip("0123456789"))
    return names


def test_fixture_tries_accept_honest_answers(oracle, golden):
    tries = fixture_tries(oracle, golden)
    assert sum(t.name.endswith("/accounts") for t in tries) == 91
    assert len(tries) == 144
    n = sum(check_accepts(oracle, t) for t in tries)
    assert n > 3000, n


def test_random_and_awkward_tries_accept_honest_answers(oracle):
    rng = np.random.default_rng(3)
    for t in random_tries(oracle) + awkward_tries(oracle):
        check_accepts(oracle, t, limit=48, rng=rng)


def test_mutations_are_never_accepted(oracle, golden):
    rng = np.random.default_rng(5)
    names = set()
    tries = random_tries(oracle) + awkward_tries(oracle) + [t for t in fixture_tries(oracle, golden) if len(t.kv) >= 6][:20]
    for t in tries:
        names |= check_mutations(oracle, t, rng)
    assert names >= {"drop-first", "drop-middle", "drop-last", "add-inside", "value-byte", "swap", "duplicate", "below-origin",
                     "empty-value", "empty-answer", "whole-truncated", "drop-node", "node-byte", "other-origin-proof", "wrong-root"}


@pytest.mark.parametrize("shape", ["empty", "single", "two"])
def test_tiny_tries(oracle, shape):
    t = next(t for t in awkward_tries(oracle) if t.name == shape)
    kc = oracle.keccak256
    assert verify_range(kc, [], t.root, bytes(32), list(t.kv), True) == (1, False)
    assert verify_range(kc, t.serve(bytes(32), 9)[1], t.root, bytes(32), list(t.kv), False) == (1, False)
    if t.kv:
        k = t.keys[0]
        assert verify_range(kc, t.serve(k, 1)[1], t.root, k, t.kv[:1], False) == (1, len(t.kv) > 1)
        assert verify_range(kc, t.serve(key_after(k), 1)[1], t.root, key_after(k), t.kv[1:2], False) == (1, False)
        assert verify_range(kc, t.serve(bytes(32), 9)[1], t.root, bytes(32), [], False)[0] != 1
    else:
        assert verify_range(kc, [], t.root, bytes(32), [(FF32, b"\x01")], False) == (0, False)


def test_edges_that_leave_the_trie(oracle):
    """an origin whose path ends at an empty branch slot, inside a diverging leaf's path and inside a diverging extension's"""
    rng = np.random.default_rng(9)
    head = bytes(rng.integers(0, 256, 29, dtype=np.uint8))
    kv = [(bytes([0x10]) + head + b"\x00\x01", b"\x01" * 40), (bytes([0x10]) + head + b"\x00\x02", b"\x02" * 40),
          (bytes([0x80]) + bytes(31), b"\x03" * 40), (bytes([0xc0]) + bytes(31), b"\x04" * 40)]
    t = KnownTrie(oracle, kv)
    kc = oracle.keccak256
    for origin in (bytes([0x50]) + bytes(31),                     # an empty slot of the root branch
                   bytes([0x80]) + bytes(30) + b"\x01",           # under the 0x8 leaf, after its key
                   bytes([0x7f]) + FF32[:31],                     # before the 0x8 leaf
                   bytes([0x10]) + head[:5] + FF32[:26],          # inside the extension's path, above it
                   bytes([0x10]) + bytes(31)):                    # inside the extension's path, below it
        for c in (1, 2, 4):
            ents, nodes, more = t.serve(origin, c)
            assert verify_range(kc, nodes, t.root, origin, ents, False) == (1, more), (origin.hex(), c)
