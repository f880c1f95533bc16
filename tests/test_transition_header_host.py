"""The device node decoder of the transition roots (phant_b200/csrc/transition.cuh) compiled as HOST code
(tests/hostcheck/transition_host.cpp) and held to the CPU statement's decoder (tests/transition_oracle.py) on every node of
the fixture witnesses, on crafted nodes and on mutations of them.  The product never runs this way; the -m gpu tests check the
same rules through the C ABI on the device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from resident_state_model import StateModel, change_diff, hashed_table, load_diff
from transition_oracle import decode, witness

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("transitionhost") / "libtransitionhost.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so,
                    os.path.join(HERE, "hostcheck", "transition_host.cpp")], check=True)
    L = C.CDLL(so)
    L.ht_decode.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint32)]
    return L


def device_decode(L, node):
    """the device decoder's result in the oracle's form"""
    node = bytes(node)
    path, plen, f = C.create_string_buffer(64), C.c_uint32(), (C.c_uint32 * 50)()
    k = L.ht_decode(node + bytes(64), len(node), path, C.byref(plen), f)
    if k == 0:
        return None

    def child(v):
        kind, o, n = f[2 + 3 * v], f[3 + 3 * v], f[4 + 3 * v]
        return None if kind == 0 else ("hash" if kind == 1 else "embed", node[o:o + n])

    p = tuple(path.raw[:plen.value])
    if k == 1:
        return ("leaf", p, node[f[0]:f[0] + f[1]])
    if k == 2:
        return ("ext", p, child(0))
    return ("branch", [child(v) for v in range(16)])


def fixture_nodes(oracle, golden):
    g = golden("fixture_states.json.gz")
    out = {}
    for t in g["tests"]:
        pre, post = hashed_table(oracle.keccak256, g["tables"][t["pre"]]), hashed_table(oracle.keccak256, g["tables"][t["post"]])
        m = StateModel(oracle)
        m.apply(load_diff(pre))
        for n in witness(oracle, m, change_diff(pre, post)):
            out[n] = 1
    return list(out)


def test_fixture_witness_nodes(lib, oracle, golden):
    nodes = fixture_nodes(oracle, golden)
    assert len(nodes) > 100
    for n in nodes:
        want = decode(n)
        assert want is not None
        assert device_decode(lib, n) == want


def test_crafted_and_mutated_nodes(lib, oracle, golden):
    crafted = [b"\xc0", b"\xc2\x20\x01", b"\xc3\x80\x80\x80", b"\xd1" + b"\x80" * 17, b"\xd1" + b"\x81\x01" + b"\x80" * 15,
               b"\xc4\x00\x82\x01\x02", b"\xc4\x11\xc2\x20\x01", b"\xc3\x10\xc1\x80", b"\xc2\x40\x01", b"\xc2\x01\x80",
               b"\xd3" + b"\xc2\x20\x01" + b"\x80" * 16, b"\xd2" + b"\xc2\x20\x01" + b"\x80" * 15 + b"\x01"]
    rng = np.random.default_rng(2)
    nodes = fixture_nodes(oracle, golden)
    for n in nodes[:300]:
        b = bytearray(n)
        for _ in range(3):
            m = bytearray(b)
            m[int(rng.integers(0, len(m)))] = int(rng.integers(0, 256))
            crafted.append(bytes(m))
        crafted.append(bytes(b[:-1]))
        crafted.append(bytes(b) + b"\x00")
    for n in crafted:
        assert device_decode(lib, n) == decode(n), n.hex()
