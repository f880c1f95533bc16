"""The device function of the ecrecover kernel (phant_b200/csrc/secp256k1.cuh) compiled as HOST code
(tests/hostcheck/ecrecover_host.cpp) against the oracle: the reference's vector, random inputs (recovery verifies nothing,
so ANY (hash, r, s, recid) is a meaningful case: both must agree on whether a key comes out and on the key), the limb
arithmetic against Python integers, the corner cases of the double multiplication, and every operation of the header on
the adversarial corpus of tests/secp_corpus.py (the one the device branches meet in tests/test_gpu_secp_device.py).  No GPU
involved."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import secp_corpus

HERE = os.path.dirname(os.path.abspath(__file__))
N = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141
P = 2 ** 256 - 0x1000003D1
GX = 0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798
GY = 0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8


@pytest.fixture(scope="module")
def dev(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("ech") / "libech.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so,
                    os.path.join(HERE, "hostcheck", "ecrecover_host.cpp")], check=True)
    return C.CDLL(so)


def recover(dev, h, sig):
    out = C.create_string_buffer(65)
    return out.raw if dev.host_ecrecover(bytes(h), bytes(sig), out) else None


def sig65(r, s, recid):
    return r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([recid])


def test_reference_vector(dev, golden):
    k = golden("ecrecover_kat.json")["erecover"]
    assert recover(dev, bytes.fromhex(k["hash"]), bytes.fromhex(k["sig65"])).hex() == k["pubkey65"]


def test_limb_arithmetic(dev):
    rng = np.random.default_rng(1)
    edge = [0, 1, 2, P - 1, P - 2, 2 ** 255, 0xFFFFFFFF, 2 ** 64 - 1, 2 ** 64, 2 ** 128 - 1, 2 ** 192 - 1, P - 0x1000003D1, N - 1, N, (P + 1) // 2]
    o1, o2 = C.create_string_buffer(32), C.create_string_buffer(32)

    def pick():
        return edge[int(rng.integers(0, len(edge)))] if rng.random() < 0.3 else int.from_bytes(rng.bytes(32), "big")
    for _ in range(8000):
        a, b = pick() % P, pick() % P
        dev.host_fp_mul(a.to_bytes(32, "big"), b.to_bytes(32, "big"), o1)
        assert int.from_bytes(o1.raw, "big") == a * b % P, (a, b)
        dev.host_fp_addsub(a.to_bytes(32, "big"), b.to_bytes(32, "big"), o1, o2)
        assert int.from_bytes(o1.raw, "big") == (a + b) % P and int.from_bytes(o2.raw, "big") == (a - b) % P, (a, b)
        a, b = a % N, b % N
        dev.host_sc_mul(a.to_bytes(32, "big"), b.to_bytes(32, "big"), o1)
        assert int.from_bytes(o1.raw, "big") == a * b % N, (a, b)


def test_random_inputs_agree_with_the_oracle(dev, oracle):
    rng = np.random.default_rng(2)
    outcomes = {True: 0, False: 0}
    for i in range(1500):
        r = int.from_bytes(rng.bytes(32), "big")
        s = int.from_bytes(rng.bytes(32), "big")
        kind = i % 10
        if kind == 0:
            r %= 2 ** 127   # small r: recid 2 / 3 can be valid (x = r + n < p)
        if kind == 1:
            s = [0, 1, N - 1, N, N + 1, 2 ** 256 - 1][i // 10 % 6]
        if kind == 2:
            r = [0, 1, N - 1, N, P - 1, 2 ** 256 - 1][i // 10 % 6]
        h = bytes(rng.bytes(32)) if kind != 3 else [bytes(32), b"\xff" * 32, N.to_bytes(32, "big"), (N - 1).to_bytes(32, "big")][i // 10 % 4]
        recid = int(rng.integers(0, 4)) if kind != 4 else int(rng.integers(4, 256))
        sig = sig65(r, s, recid)
        want, got = oracle.ecrecover(h, sig), recover(dev, h, sig)
        assert got == want, (r, s, recid, h.hex())
        outcomes[want is not None] += 1
    assert outcomes[True] > 300 and outcomes[False] > 300


def test_corner_cases_of_the_double_multiplication(dev, oracle):
    """R = G (the table's G + R needs the doubling branch), R = -G (G + R is the point at infinity), and u1 / u2 chosen so
    that the accumulator meets the point it is about to add"""
    rng = np.random.default_rng(4)
    for recid in (GY & 1, (GY & 1) ^ 1):          # R = G, then R = -G
        for _ in range(40):
            h, s = bytes(rng.bytes(32)), int.from_bytes(rng.bytes(32), "big") % (N - 1) + 1
            sig = sig65(GX, s, recid)
            assert recover(dev, h, sig) == oracle.ecrecover(h, sig)
    # u1 = -z/r, u2 = s/r: z = 0 -> only R is multiplied; s = r -> u2 = 1; z = -s*? ... small scalars walk through the
    # first additions where acc is still at infinity or equals a table entry
    for z, s_of_r in [(0, lambda r: r), (0, lambda r: 2 * r % N), (1, lambda r: r), (N - 1, lambda r: r), (N - 1, lambda r: (N - r) % N)]:
        for _ in range(20):
            r = int.from_bytes(rng.bytes(32), "big") % (N - 1) + 1
            s = s_of_r(r) or 1
            for recid in (0, 1):
                sig = sig65(r, s, recid)
                h = z.to_bytes(32, "big")
                assert recover(dev, h, sig) == oracle.ecrecover(h, sig), (r, s, recid, z)
    # Q at infinity: u1 G + u2 R = 0 with R = G: u1 + u2 = 0 <=> s = z (mod n)
    z = int.from_bytes(rng.bytes(32), "big") % N
    sig = sig65(GX, z, GY & 1)
    assert recover(dev, z.to_bytes(32, "big"), sig) is None and oracle.ecrecover(z.to_bytes(32, "big"), sig) is None


@pytest.mark.parametrize("op", secp_corpus.OPS)
def test_corpus_through_the_host_branch(dev, op):
    """the `#else` branches (C carries, the portable schoolbook mul_wide, fp_reduce's C fold, the __int128 mac) on the
    adversarial corpus that tests/test_gpu_secp_device.py runs through the device branches: every output equal to Python's
    value, canonical, carry words 0 or 1"""
    in_w, out_w, n_ops = C.c_int(), C.c_int(), C.c_int()
    dev.secp_check_layout(C.byref(in_w), C.byref(out_w), C.byref(n_ops))
    assert (in_w.value, out_w.value, n_ops.value) == (secp_corpus.IN_WORDS, secp_corpus.OUT_WORDS, len(secp_corpus.OPS))

    def run(code, inp):
        inp = np.ascontiguousarray(inp)
        out = np.zeros((inp.shape[0], secp_corpus.OUT_WORDS), np.uint64)
        assert dev.secp_check_run(code, C.c_void_p(inp.ctypes.data), C.c_void_p(out.ctypes.data), C.c_uint64(inp.shape[0])) == 0
        return out
    assert secp_corpus.check(run, op) == len(secp_corpus.cases(op))

