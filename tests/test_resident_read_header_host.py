"""The device per-key reads of the resident world state (phant_b200/csrc/resident_read.cuh) compiled as HOST code
(tests/hostcheck/resident_read_host.cpp) and held to the Python model at every root a journal reaches.  Block sequences go
through tests/resident_state_model.py; each apply's undo record is tests/resident_state_undo.py's inverse, laid out as the
device lays it out (accounts sorted by key, slots by (record account, slot key), the accounts' old storage roots from the
model).  Every read at every `back` must equal the model's snapshot of that block, storage roots included.  The -m gpu tests
check the same reads through the C ABI on the device."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from resident_state_model import CLEAR, DELETE, ZERO32, Diff, StateModel
from resident_state_undo import inverse, snapshot

HERE = os.path.dirname(os.path.abspath(__file__))


class RdRec(C.Structure):
    _fields_ = [(f, C.c_void_p) for f in ("akeys", "aflags", "nonce", "bal", "code", "sroot", "sacc", "skeys", "svals")] + \
               [("na", C.c_uint32), ("ms", C.c_uint32)]


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("residentreadhost") / "libresidentreadhost.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so,
                    os.path.join(HERE, "hostcheck", "resident_read_host.cpp")], check=True)
    L = C.CDLL(so)
    L.hr_account.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32, C.c_char_p, C.POINTER(C.c_uint64), C.c_void_p]
    L.hr_slot.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_uint32, C.c_char_p, C.c_char_p, C.c_void_p]
    return L


def cat(xs, width):
    return np.frombuffer(b"".join(xs) + bytes(width), np.uint8).copy()  # slack behind the last entry, as on the device


def tables(m):
    """the model's current state as the device holds it: the account trie's rows (key, arena offset, length) and arena of
    account bodies, and the slot table sorted by (account key, slot key)"""
    ks = sorted(m.acc)
    krows = np.zeros((max(len(ks), 1), 80), np.uint8)
    bodies, off = [], 0
    for i, k in enumerate(ks):
        b = m.leaf(k)
        krows[i, :32] = np.frombuffer(k, np.uint8)
        krows[i, 32:40] = np.frombuffer(np.uint64(off).tobytes(), np.uint8)
        krows[i, 40:44] = np.frombuffer(np.uint32(len(b)).tobytes(), np.uint8)
        bodies.append(b)
        off += len(b)
    rows = sorted((k, sk, v) for k in ks for sk, v in m.acc[k].storage.items())
    srows = np.zeros((max(len(rows), 1), 96), np.uint8)
    for i, (k, sk, v) in enumerate(rows):
        srows[i] = np.frombuffer(k + sk + v, np.uint8)
    return krows, len(ks), cat(bodies, 64), srows, len(rows)


def record(m, d):
    """the undo record of applying d to m (before it applies), in the device's layout: numpy arrays"""
    inv = inverse(m, d)
    order = sorted(range(len(inv.accounts)), key=lambda i: inv.accounts[i][0])
    pos = {i: p for p, i in enumerate(order)}
    acc = [inv.accounts[i] for i in order]
    slots = sorted((pos[ai], sk, v) for ai, sk, v in inv.slots)
    sroot = [ZERO32 if f & DELETE else m.storage_root(k) for k, f, _, _, _ in acc]
    r = dict(akeys=cat([a[0] for a in acc], 32), aflags=np.array([a[1] for a in acc] + [0], np.uint8),
             nonce=np.array([a[2] for a in acc] + [0], np.uint64), bal=cat([a[3] for a in acc], 32), code=cat([a[4] for a in acc], 32),
             sroot=cat(sroot, 32), sacc=np.array([s[0] for s in slots] + [0], np.uint32), skeys=cat([s[1] for s in slots], 32),
             svals=cat([s[2] for s in slots], 32))
    return r, len(acc), len(slots)


class Reader:
    def __init__(self, oracle):
        self.m = StateModel(oracle)
        self.journal = []  # (record arrays, na, ms), oldest first
        self.hist = [self.m.copy()]

    def apply(self, d):
        self.journal.append(record(self.m, d))
        self.m.apply(d)
        self.hist.append(self.m.copy())

    def check(self, L, akeys, slots):
        """every key at every back against the history"""
        krows, n, arena, srows, nS = tables(self.m)
        nonce, out = C.c_uint64(), np.zeros(96, np.uint8)
        for back in range(len(self.journal) + 1):
            win = self.journal[len(self.journal) - back:]
            recs = (RdRec * max(back, 1))(*[RdRec(*[r[f].ctypes.data for f, _ in RdRec._fields_[:9]], na, ms) for r, na, ms in win])
            want_m = self.hist[len(self.hist) - 1 - back]
            want = snapshot(want_m)
            for k in akeys:
                st = L.hr_account(krows.ctypes.data, n, arena.ctypes.data, recs, back, k, C.byref(nonce), out.ctypes.data)
                if k in want:
                    nn, bal, ch, _ = want[k]
                    assert st == 1, (back, k.hex())
                    assert (nonce.value, out[:32].tobytes(), out[32:64].tobytes(), out[64:].tobytes()) == \
                        (nn, bal, want_m.storage_root(k), ch), (back, k.hex())
                else:
                    assert st == 2 and nonce.value == 0 and not out.any(), (back, k.hex())
            for k, sk in slots:
                st = L.hr_slot(srows.ctypes.data, nS, recs, back, k, sk, out.ctypes.data)
                v = want[k][3].get(sk, ZERO32) if k in want else ZERO32
                assert (st, out[:32].tobytes()) == ((1, v) if v != ZERO32 else (2, ZERO32)), (back, k.hex(), sk.hex())


def rk(rng):
    return rng.bytes(32)


def val(rng):
    return bytes(31) + bytes([int(rng.integers(1, 256))]) if rng.random() < 0.5 else rng.bytes(32)


def test_scripted_sequence(lib, oracle):
    """a destroy then a re-create across blocks, CLEAR_STORAGE then a write in a newer record, a slot written only in a newer
    record, and empty applies"""
    rng = np.random.default_rng(1)
    r = Reader(oracle)
    a, b, c = rk(rng), rk(rng), rk(rng)
    s = [rk(rng) for _ in range(6)]
    f = lambda n: (n, (n * 7).to_bytes(32, "big"), rk(rng))  # noqa: E731
    r.apply(Diff([(a, 0) + f(1), (b, 0) + f(2)], [(0, s[0], val(rng)), (0, s[1], val(rng)), (1, s[2], val(rng))]))
    r.apply(Diff())                                                                      # empty
    r.apply(Diff([(a, DELETE, 0, ZERO32, ZERO32)]))                                      # destroy
    r.apply(Diff([(a, 0) + f(3)], [(0, s[3], val(rng))]))                                # re-create
    r.apply(Diff([(b, CLEAR) + f(4)], [(0, s[4], val(rng))]))                            # clear, one write
    r.apply(Diff([(b, 0) + f(5)], [(0, s[2], val(rng)), (0, s[5], val(rng)), (0, s[4], ZERO32)]))  # newer writes
    r.apply(Diff([(c, 0) + f(6)], [(0, s[0], val(rng))]))                                # a slot written only here
    r.apply(Diff([(c, DELETE, 0, ZERO32, ZERO32), (a, CLEAR) + f(7)]))                   # destroy and clear in one apply
    r.apply(Diff())
    r.apply(Diff([(c, 0) + f(8)]))
    ghost = rk(rng)
    r.check(lib, [a, b, c, ghost], [(k, sk) for k in (a, b, c, ghost) for sk in s])


@pytest.mark.parametrize("seed", range(6))
def test_random_sequences(lib, oracle, seed):
    rng = np.random.default_rng(100 + seed)
    r = Reader(oracle)
    keys = [rk(rng) for _ in range(10)]
    skeys = [rk(rng) for _ in range(8)]
    for _ in range(12):
        if rng.random() < 0.1:
            r.apply(Diff())
            continue
        accounts, slots = [], []
        for k in rng.choice(len(keys), int(rng.integers(1, 6)), replace=False):
            x = rng.random()
            flags = DELETE if x < 0.15 else CLEAR if x < 0.3 else 0
            accounts.append((keys[k], flags, int(rng.integers(0, 1 << 40)), val(rng), rk(rng)))
            if flags & DELETE:
                continue
            for sk in rng.choice(len(skeys), int(rng.integers(0, 5)), replace=False):
                slots.append((len(accounts) - 1, skeys[sk], ZERO32 if rng.random() < 0.25 else val(rng)))
        r.apply(Diff(accounts, slots))
    r.check(lib, keys + [rk(rng)], [(k, sk) for k in keys for sk in skeys])
