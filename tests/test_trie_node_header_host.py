"""The device walk by nibble path behind the resident state's trie nodes (phant_b200/csrc/proof_chain.cuh, pc_node_at)
compiled as HOST code (tests/hostcheck/trie_node_host.cpp) and held to the CPU statement (tests/trie_node_model.py): on the
fixture tries and on random tries with extensions, embedded storage leaves and pairs sharing 62 and 63 nibbles, every node's
own path is served with that node, and every other path -- inside an extension's or a leaf's path, below a leaf, at an
embedded node, diverging at every depth, of length 64 -- has none, nor has any path of the empty trie.  The node set is
what the GPU walks: the served nodes, each once, ordered by digest."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from resident_state_model import StateModel, hashed_table, load_diff
from test_trie_node_model import random_trie
from trie_node_model import nibbles, pack, probe_paths, served, storage_value, trie_nodes

HERE = os.path.dirname(os.path.abspath(__file__))
EMPTY = bytes.fromhex("56e81f171bcc55a6ff8345e692c0f86e5b48e01b996cadc001622fb5e363b421")


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("trienodehost") / "libtrienodehost.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so,
                    os.path.join(HERE, "hostcheck", "trie_node_host.cpp")], check=True)
    L = C.CDLL(so)
    L.hp_node_at.argtypes = [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 4 + [C.c_uint32] + [C.c_void_p] * 2
    L.hp_node_at.restype = None
    return L


def check_trie(L, oracle, kv, extra=()):
    """every probe path around kv's keys (and `extra`): status 1 with the statement's node exactly where it serves one.
    Returns the counts of (paths served, embedded nodes probed, 64-nibble paths served)."""
    root, nodes = trie_nodes(oracle.keccak256, kv)
    s = served(nodes)
    order = sorted(s.values(), key=oracle.keccak256)
    index = {e: i for i, e in enumerate(order)}
    off = np.zeros(len(order) + 1, np.uint64)
    off[1:] = np.cumsum([len(e) for e in order])
    data = np.frombuffer(b"".join(order) + bytes(64), np.uint8).copy()
    dig = np.frombuffer(b"".join(oracle.keccak256(e) for e in order) + bytes(32), np.uint8).copy()
    rng = np.random.default_rng(len(kv))
    paths = probe_paths(kv, rng) + [tuple(p) for p in extra]
    packed = [pack(p) for p in paths]
    pa = np.frombuffer(b"".join(b for b, _ in packed), np.uint8).copy()
    pl = np.array([n for _, n in packed], np.uint8)
    status, idx = np.zeros(len(paths), np.uint8), np.zeros(len(paths), np.uint32)
    rb, eb = np.frombuffer(root, np.uint8).copy(), np.frombuffer(EMPTY, np.uint8).copy()
    L.hp_node_at(data.ctypes.data, off.ctypes.data, dig.ctypes.data, len(order), rb.ctypes.data, eb.ctypes.data, pa.ctypes.data,
                 pl.ctypes.data, len(paths), status.ctypes.data, idx.ctypes.data)
    for i, p in enumerate(paths):
        if p in s:
            assert status[i] == 1 and int(idx[i]) == index[s[p]], p
        else:
            assert status[i] == 2, p
    return sum(1 for p in paths if p in s), sum(1 for p in paths if p in nodes and p not in s), sum(1 for p in s if len(p) == 64)


def test_fixture_tries(lib, oracle, golden):
    g = golden("fixture_states.json.gz")
    seen = 0
    for name in sorted(g["tables"]):
        m = StateModel(oracle)
        m.apply(load_diff(hashed_table(oracle.keccak256, g["tables"][name])))
        check_trie(lib, oracle, {k: m.leaf(k) for k in m.acc})
        for a in m.acc.values():
            if a.storage:
                check_trie(lib, oracle, {sk: storage_value(v) for sk, v in a.storage.items()})
                seen += 1
    assert seen > 20


def test_random_tries(lib, oracle):
    rng = np.random.default_rng(11)
    embedded = deep = 0
    for trial in range(30):
        _, e, d = check_trie(lib, oracle, random_trie(rng, int(rng.integers(1, 200)), trial % 3))
        embedded += e
        deep += d
    assert embedded > 0 and deep > 0


def test_single_leaf_and_empty_trie(lib, oracle):
    rng = np.random.default_rng(2)
    k = rng.bytes(32)
    served_n, _, _ = check_trie(lib, oracle, {k: rng.bytes(40)})
    assert served_n == 1  # the root leaf only: every deeper prefix ends inside its path
    check_trie(lib, oracle, {}, extra=[(), nibbles(k)[:5], nibbles(k)])
