"""The device per-range rules of the range-proof check (phant_b200/csrc/range_proof.cuh) compiled as HOST code
(tests/hostcheck/range_proof_host.cpp) and held to the CPU statement (tests/range_proof_oracle.py) over the corpus of
tests/range_proof_corpus.py: the entry checks of every honest answer and every mutation, the upper edge key, and the
inside / above test of every prefix of every key of each trie against each answer's edges.  The product never runs this way;
the -m gpu tests check the same rules through the C ABI on the device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from range_proof_corpus import accept_cases, awkward_tries, fixture_tries, mutation_cases, random_tries
from range_proof_oracle import entries_ok, last_key
from transition_oracle import nibbles

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("rangeproofhost") / "librangeproofhost.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-o", so, os.path.join(HERE, "hostcheck", "range_proof_host.cpp")],
                   check=True)
    L = C.CDLL(so)
    L.hr_entries_ok.argtypes = [C.c_char_p, C.c_void_p, C.c_uint32, C.c_char_p, C.c_int]
    L.hr_last.argtypes = [C.c_char_p, C.c_char_p]
    L.hr_classify.argtypes = [C.c_char_p, C.c_uint32, C.c_char_p, C.c_char_p]
    return L


def device_entries_ok(L, entries, origin, whole):
    keys = b"".join(k for k, _ in entries) or bytes(32)
    off = np.zeros(len(entries) + 1, np.uint64)
    off[1:] = np.cumsum([len(v) for _, v in entries])
    return bool(L.hr_entries_ok(keys, off.ctypes.data, len(entries), origin, int(whole)))


def device_last(L, entries):
    out = C.create_string_buffer(32)
    L.hr_last(entries[-1][0] if entries else None, out)
    return out.raw


def prefix_key(key, depth):
    """the key's first `depth` nibbles, zero after: how a stub's prefix is held"""
    n = nibbles(key)[:depth] + (0,) * (64 - depth)
    return bytes((n[i] << 4) | n[i + 1] for i in range(0, 64, 2))


def answers(oracle, golden):
    rng = np.random.default_rng(4)
    out = []
    for t in fixture_tries(oracle, golden)[::3] + random_tries(oracle) + awkward_tries(oracle):
        out += [(t, o, e, w) for o, e, _, w, _ in accept_cases(t, limit=12, rng=rng)]
        out += [(t, c[2], c[3], c[5]) for c in mutation_cases(t, rng)]
    return out


def test_entry_checks_and_last(lib, oracle, golden):
    n_bad = 0
    for t, origin, ents, whole in answers(oracle, golden):
        want = entries_ok(ents, origin, whole)
        assert device_entries_ok(lib, ents, origin, whole) == want, (t.name, origin.hex())
        assert device_last(lib, ents) == last_key(ents)
        n_bad += not want
    assert n_bad > 50


def test_inside_and_above(lib, oracle, golden):
    rng = np.random.default_rng(8)
    n = 0
    for t, origin, ents, whole in answers(oracle, golden):
        if whole or not entries_ok(ents, origin, whole) or not t.keys:
            continue
        last = last_key(ents)
        lo, hi = nibbles(origin), nibbles(last)
        keys = [t.keys[int(i)] for i in rng.choice(len(t.keys), min(len(t.keys), 6), replace=False)] + [origin, last]
        for k in keys:
            for depth in sorted({0, 1, 2, 63, 64} | {int(x) for x in rng.integers(0, 65, 4)}):
                p = prefix_key(k, depth)
                pn = nibbles(p)[:depth]
                first, end = pn + (0,) * (64 - depth), pn + (15,) * (64 - depth)
                want = (1 if lo <= first and end <= hi else 0) | (2 if first > hi else 0)
                assert lib.hr_classify(p, depth, origin, last) == want, (k.hex(), depth, origin.hex(), last.hex())
                n += 1
    assert n > 20000
