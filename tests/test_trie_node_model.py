"""The CPU statement of the trie nodes served by path (tests/trie_node_model.py) pinned to the C oracle: its root is
oracle_trie_root's, and for every key the oracle's proof chain is exactly the statement's served nodes at the key's prefixes,
root first -- on every fixture trie and on random tries with extensions, embedded leaves and keys sharing 62 or 63 nibbles.
py_mptize gives a third root."""
import numpy as np

from helpers import py_mptize, rlp_str
from resident_state_model import StateModel, hashed_table, load_diff
from trie_node_model import nibbles, served, storage_value, trie_nodes


def check(oracle, kv):
    root, nodes = trie_nodes(oracle.keccak256, kv)
    items = sorted(kv.items())
    if not items:
        assert root == oracle.keccak256(b"\x80") and nodes == {}
        return
    t = oracle.trie(items)
    assert root == t.root() == py_mptize(oracle.keccak256, items)
    s = served(nodes)
    assert all(oracle.keccak256(e) == root for p, e in s.items() if p == ())
    for k in kv:
        n = nibbles(k)
        assert t.prove(k) == [s[n[:d]] for d in range(65) if n[:d] in s], k.hex()
    return nodes


def random_trie(rng, n, shared):
    kv = {}
    for _ in range(n):
        k = bytearray(rng.bytes(32))
        if shared == 1:
            k[:28] = b"\x42" * 28  # extensions over long shared prefixes
        v = bytes([int(rng.integers(1, 0x80))]) if rng.integers(0, 2) else rng.bytes(int(rng.integers(1, 40)))
        kv[bytes(k)] = storage_value(v) if shared == 2 else v
    if shared == 2:  # pairs sharing 62 and 63 nibbles, with 1-byte values: embedded leaves
        for _ in range(4):
            b = rng.bytes(31)
            kv[b + b"\x10"], kv[b + b"\x11"] = rlp_str(b"\x05"), rlp_str(b"\x06")
            kv[b + b"\x20"] = rlp_str(rng.bytes(32))
            kv[b + b"\x30"], kv[b + b"\x31"] = rlp_str(rng.bytes(32)), rlp_str(b"\x07")  # a hashed leaf at depth 64
    return kv


def test_fixture_tries(oracle, golden):
    g = golden("fixture_states.json.gz")
    seen = 0
    for name in sorted(g["tables"]):
        m = StateModel(oracle)
        m.apply(load_diff(hashed_table(oracle.keccak256, g["tables"][name])))
        check(oracle, {k: m.leaf(k) for k in m.acc})
        for a in m.acc.values():
            if a.storage:
                check(oracle, {sk: rlp_str(v.lstrip(b"\x00")) for sk, v in a.storage.items()})
                seen += 1
    assert seen > 20


def test_random_tries(oracle):
    rng = np.random.default_rng(5)
    embedded = deep = 0
    for trial in range(30):
        nodes = check(oracle, random_trie(rng, int(rng.integers(1, 200)), trial % 3))
        embedded += sum(1 for p, e in nodes.items() if p and len(e) < 32)
        deep += sum(1 for p in served(nodes) if len(p) == 64)
    assert embedded > 0 and deep > 0
    check(oracle, {})
