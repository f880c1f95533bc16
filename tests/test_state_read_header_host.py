"""The device decoders of pre-state reads (phant_b200/csrc/state_read.cuh) compiled as HOST code
(tests/hostcheck/state_read_host.cpp) and held to the test decoders of tests/state_read_oracle.py on valid account bodies
and slot values and on every mutation class of DESIGN.md "P: pre-state reads".  The product never runs this way; the -m gpu
tests check the same rules through the C ABI on the device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import rlp_list, rlp_str
from state_read_oracle import decode_account, decode_slot

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("statereadhost") / "libstatereadhost.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so,
                    os.path.join(HERE, "hostcheck", "state_read_host.cpp")], check=True)
    L = C.CDLL(so)
    L.hs_decode_account.argtypes = [C.c_char_p, C.c_uint32, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    L.hs_decode_slot.argtypes = [C.c_char_p, C.c_uint32, C.POINTER(C.c_uint32)]
    return L


def device_account(L, body):
    buf = bytes(body) + bytes(64)  # the device buffers carry slack behind every node
    nonce, f = C.c_uint64(), (C.c_uint32 * 4)()
    if not L.hs_decode_account(buf, len(body), C.byref(nonce), f):
        return None
    b = bytes(body)
    return nonce.value, b[f[0]:f[0] + f[1]], b[f[2]:f[2] + 32], b[f[3]:f[3] + 32]


def device_slot(L, payload):
    f = (C.c_uint32 * 2)()
    if not L.hs_decode_slot(bytes(payload) + bytes(64), len(payload), f):
        return None
    return bytes(payload)[f[0]:f[0] + f[1]]


def trim(x, n):
    return x.to_bytes(n, "big").lstrip(b"\x00")


def account(nonce, bal, root=None, code=None, rng=None):
    root = root if root is not None else bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    code = code if code is not None else bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    return rlp_list([rlp_str(trim(nonce, 8)), rlp_str(trim(bal, 32)), rlp_str(root), rlp_str(code)])


def valid_accounts(rng):
    nonces = [0, 1, 0x7F, 0x80, 0xFF, 0x100, 2 ** 56, 2 ** 64 - 1] + [int(rng.integers(0, 2 ** 63)) for _ in range(8)]
    bals = [0, 1, 0x7F, 0x80, 2 ** 64, 2 ** 255, 2 ** 256 - 1] + [int.from_bytes(rng.bytes(int(rng.integers(1, 33))), "big") for _ in range(9)]
    return [account(n, b, rng=rng) for n, b in zip(nonces, bals)]


def header_mutations(body):
    """every byte flipped (two ways), truncation by 1..n bytes, each length byte of the top list +-1, trailing bytes"""
    out = []
    for i in range(len(body)):
        for x in (0x01, 0xFF):
            m = bytearray(body); m[i] ^= x; out.append(bytes(m))
    out += [body[:len(body) - k] for k in range(1, len(body) + 1)]
    for i in range(min(2, len(body))):
        for d in (-1, 1):
            m = bytearray(body); m[i] = (m[i] + d) & 0xFF; out.append(bytes(m))
    out += [body + b"\x00", body + b"\x80"]
    return out


def structural_account_mutations(rng):
    r32, c32 = bytes(range(32)), bytes(32)
    bad_items = [
        [b"\x00", rlp_str(b"\x01"), rlp_str(r32), rlp_str(c32)],                 # nonce 0x00: a leading zero
        [rlp_str(b"\x00\x05"), rlp_str(b"\x01"), rlp_str(r32), rlp_str(c32)],    # nonce with a leading zero
        [b"\x05", rlp_str(b"\x00\x01"), rlp_str(r32), rlp_str(c32)],             # balance with a leading zero
        [b"\x05", b"\x00", rlp_str(r32), rlp_str(c32)],                           # balance 0x00
        [rlp_str(b"\x01" * 9), rlp_str(b"\x01"), rlp_str(r32), rlp_str(c32)],    # 9-byte nonce
        [b"\x05", rlp_str(b"\x01" * 33), rlp_str(r32), rlp_str(c32)],            # 33-byte balance
        [b"\x05", rlp_str(b"\x01"), rlp_str(r32[:31]), rlp_str(c32)],            # 31-byte root
        [b"\x05", rlp_str(b"\x01"), rlp_str(r32 + b"\x01"), rlp_str(c32)],       # 33-byte root
        [b"\x05", rlp_str(b"\x01"), rlp_str(r32), rlp_str(c32[:31])],            # 31-byte code hash
        [b"\x05", rlp_str(b"\x01"), rlp_str(r32), rlp_str(c32 + b"\x00")],       # 33-byte code hash
        [b"\x05", rlp_list([b"\x01"]), rlp_str(r32), rlp_str(c32)],               # a list where a string belongs
        [rlp_list([]), rlp_str(b"\x01"), rlp_str(r32), rlp_str(c32)],
        [b"\x05", rlp_str(b"\x01"), rlp_list([rlp_str(r32)]), rlp_str(c32)],
        [b"\x05", rlp_str(r32), rlp_str(c32)],                                     # 3 items
        [b"\x05", rlp_str(b"\x01"), rlp_str(r32), rlp_str(c32), b"\x01"],         # 5 items
        [b"\xb8\x01\x05", rlp_str(b"\x01"), rlp_str(r32), rlp_str(c32)],          # long-form header for a 1-byte payload
        [b"\x81\x05", rlp_str(b"\x01"), rlp_str(r32), rlp_str(c32)],              # single byte < 0x80 not encoded as itself
        [b"\x05", b"\xb8\x01\x01", rlp_str(r32), rlp_str(c32)],
        [b"\x05", rlp_str(b"\x01"), b"\xb8\x20" + r32, rlp_str(c32)],             # long form for a 32-byte string
        [b"\x05", rlp_str(b"\x01"), rlp_str(r32), b"\xb8\x20" + c32],
    ]
    out = [rlp_list(items) for items in bad_items]
    body = rlp_list([b"\x05", rlp_str(b"\x01"), rlp_str(r32), rlp_str(c32)])
    out.append(b"\xf9\x00" + body[1:])            # long-form list header with a leading zero length byte
    out.append(b"\xb8" + body[1:])                # a string, not a list
    out.append(rlp_str(body))                     # the whole body wrapped as a string
    return out


def valid_slots():
    out = []
    for n in range(1, 33):
        for first in (0x01, 0x7F, 0x80, 0xFF):
            out.append(rlp_str(bytes([first]) + bytes(range(n - 1))))
    return out


def slot_mutations(rng):
    out = [b"", b"\x80", b"\x00", rlp_str(b"\x00\x01"), rlp_str(b"\x00" * 32), rlp_str(b"\x01" * 33), b"\x81\x05", b"\xb8\x01\x80",
           b"\xb8\x20" + b"\x01" * 32, b"\xc1\x01", rlp_list([rlp_str(b"\x01" * 32)]), b"\x05\x00", rlp_str(b"\x01" * 32) + b"\x00"]
    for v in (rlp_str(b"\x2a"), rlp_str(b"\x80" + bytes(range(31))), rlp_str(b"\x01\x02\x03")):
        out += header_mutations(v)
    return out


def test_accounts_valid_and_mutated(lib):
    rng = np.random.default_rng(11)
    n_ok = n_bad = 0
    cases = valid_accounts(rng)
    for body in valid_accounts(rng)[:6]:
        cases += header_mutations(body)
        # the length byte of each item +-1
        pos = 2
        while pos < len(body):
            t = body[pos]
            for d in (-1, 1):
                m = bytearray(body); m[pos] = (t + d) & 0xFF; cases.append(bytes(m))
            pos += 1 if t < 0x80 else 1 + (t - 0x80)
    cases += structural_account_mutations(rng)
    for body in cases:
        want = decode_account(body)
        got = device_account(lib, body)
        assert got == want, (body.hex(), got, want)
        n_ok += want is not None
        n_bad += want is None
    assert n_ok >= 16 and n_bad >= 500, (n_ok, n_bad)


def test_slot_values_valid_and_mutated(lib):
    rng = np.random.default_rng(12)
    cases = valid_slots() + slot_mutations(rng)
    n_ok = n_bad = 0
    for v in cases:
        want = decode_slot(v)
        got = device_slot(lib, v)
        assert got == want, (v.hex(), got, want)
        n_ok += want is not None
        n_bad += want is None
    assert n_ok >= 128 and n_bad >= 60, (n_ok, n_bad)
    assert device_slot(lib, b"\x80") is None and device_slot(lib, b"\x00") is None  # a zero value is never stored
