"""The device rules of the snap range answers (phant_b200/csrc/snap_range.cuh) compiled as HOST code and run as one whole
call's entries (tests/hostcheck/snap_range_host.cpp: windows, sizes, scan, cuts, fill), held to the CPU statement
(tests/snap_serve_model.py): every cut, every served account and every slim and slot body, byte for byte.  Budgets 0, 1, 36,
37, exactly at an entry boundary and either side of it, 2 MiB and 2^63; limits at a key, between keys, below the origin and
above every key; storage requests whose first account is cut, that stop at the first slot of a later account, that meet
their budget exactly at an account's end, and that hold absent accounts or accounts without storage in the middle; slim
bodies with the empty root and code, zero nonce and balance, and a 32-byte balance.  Three mutants of the header -- `>=` in
place of `>` in the soft cut, the hard limit dropped, the limit applied to every account -- must each fail a case."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from resident_state_model import Diff, StateModel
from snap_serve_model import EMPTY_CODE, FF, ZERO, Prover, account_answer, slim, slot_body, storage_answer
from test_resident_read_header_host import tables

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "phant_b200", "csrc")
MUTANTS = {"soft >=": ("if (x[mid] - x[0] > bytes) b = mid;", "if (x[mid] - x[0] >= bytes) b = mid;"),
           "no hard limit": ("const uint64_t hard = snp_hard(bytes);", "const uint64_t hard = ~0ull;"),
           "limit everywhere": ("k ? ff : limit, lo[k], run[k]", "limit, lo[k], run[k]")}


def build(out_dir, header=None):
    inc = [os.path.join(ROOT, "include"), CSRC]
    if header is not None:
        with open(os.path.join(out_dir, "snap_range.cuh"), "w") as f:
            f.write(header)
        inc.insert(0, str(out_dir))
    so = os.path.join(out_dir, "libsnaprangehost.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so] + [f"-I{d}" for d in inc] +
                   [os.path.join(HERE, "hostcheck", "snap_range_host.cpp")], check=True)
    L = C.CDLL(so)
    vp = C.c_void_p
    L.hs_snap.argtypes = [vp, C.c_uint32, vp, vp, C.c_uint32, C.c_uint32, vp, vp, vp, C.c_uint32, vp, vp, vp, vp, vp, C.c_uint64,
                          C.c_uint64, vp, vp, vp, vp, vp, vp]
    return L


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return build(tmp_path_factory.mktemp("snaprangehost"))


def add(k, d):
    return ((int.from_bytes(k, "big") + d) % (1 << 256)).to_bytes(32, "big")


def run(L, m, ar, sr):
    """the harness's answers as the model states them: ([(key, body)] per account request, [[(key, body)] per served account]
    per storage request)"""
    krows, nK, arena, srows, nS = tables(m)
    cat = lambda xs: np.frombuffer(b"".join(xs) or bytes(32), np.uint8).copy()  # noqa: E731
    n, mm = len(ar), len(sr)
    first = np.zeros(mm + 1, np.uint64)
    first[1:] = np.cumsum([len(r[0]) for r in sr])
    M = int(first[mm])
    cap = 1 << 16
    ent, served, proved = np.zeros(n + M + 1, np.uint64), np.zeros(mm + 1, np.uint64), np.zeros(mm + 1, np.uint32)
    keys, boff, bodies = np.zeros(32 * cap, np.uint8), np.zeros(cap + 1, np.uint64), np.zeros(120 * cap, np.uint8)
    keep = [cat([r[0] for r in ar]), cat([r[1] for r in ar]), np.array([r[2] for r in ar] + [0], np.uint64),
            cat([a for r in sr for a in r[0]]), cat([r[1] for r in sr]), cat([r[2] for r in sr]), np.array([r[3] for r in sr] + [0], np.uint64)]
    ao, al, ab, sa, so, sl, sb = (x.ctypes.data for x in keep)
    rc = L.hs_snap(krows.ctypes.data, nK, arena.ctypes.data, srows.ctypes.data, nS, n, ao, al, ab, mm, first.ctypes.data, sa, so, sl, sb,
                   cap, bodies.size, ent.ctypes.data, served.ctypes.data, proved.ctypes.data, keys.ctypes.data, boff.ctypes.data,
                   bodies.ctypes.data)
    assert rc == 0
    e, seg = 0, 0

    def take(k):
        nonlocal e
        out = [(keys[32 * i:32 * i + 32].tobytes(), bodies[int(boff[i]):int(boff[i + 1])].tobytes()) for i in range(e, e + k)]
        e += k
        return out
    accounts = [take(int(ent[r])) for r in range(n)]
    seg = n
    slots = []
    for q in range(mm):
        lists = [take(int(ent[seg + k])) for k in range(int(first[q + 1] - first[q]))]
        slots.append(lists[:int(served[q])])
        assert all(not x for x in lists[int(served[q]):])
        seg += len(lists)
    return accounts, slots


def mismatches(L, m, ar, sr):
    pv = Prover(None, m)
    pv.chain = lambda owner, key: []  # the header holds the entries; proofs are the device's node set's (GPU tests)
    got_a, got_s = run(L, m, ar, sr)
    bad = [("account", i) for i, r in enumerate(ar) if got_a[i] != account_answer(m, pv, *r)[0]]
    bad += [("storage", j) for j, r in enumerate(sr) if got_s[j] != storage_answer(m, pv, *r)[0]]
    return bad


def state(oracle):
    """accounts with the empty root and code, zero nonce and balance, a 32-byte balance, and a few with storage: one with
    40 slots of mixed widths, one with 3 one-byte slots, one with a single 32-byte slot"""
    rng = np.random.default_rng(81)
    d = Diff()
    d.accounts.append((b"\x10" * 32, 0, 0, bytes(32), EMPTY_CODE))                       # the 37-byte entry
    d.accounts.append((b"\x20" * 32, 0, (1 << 64) - 1, b"\xff" * 32, rng.bytes(32)))      # the widest
    d.accounts += [(rng.bytes(32), 0, int(rng.integers(0, 300)), int(rng.integers(0, 1 << 40)).to_bytes(32, "big"), rng.bytes(32))
                   for _ in range(60)]
    for i, n in ((2, 40), (3, 3), (4, 1)):
        for j in range(n):
            v = bytes([int(rng.integers(1, 256))]).rjust(32, b"\x00") if n != 40 else rng.bytes(int(rng.integers(1, 33))).rjust(32, b"\x01")
            d.slots.append((i, rng.bytes(32), v))
    m = StateModel(oracle)
    m.apply(d)
    return m


def cases(m):
    keys = sorted(m.acc)
    sizes = [32 + len(slim(m, k)) for k in keys]
    at = sum(sizes[:5])
    ar = [(ZERO, FF, b) for b in (0, 1, 36, 37, at - 1, at, at + 1, 2 << 20, 1 << 63)]
    ar += [(keys[3], keys[7], 1 << 20), (keys[3], add(keys[7], -1), 1 << 20), (keys[3], add(keys[7], 1), 1 << 20), (keys[9], keys[2], 1000),
           (keys[3], FF, 1 << 20), (add(keys[-1], 1), FF, 1000), (keys[-1], FF, 0), (add(keys[5], 1), FF, 37 * 3)]
    rich = sorted((k for k in keys if m.acc[k].storage), key=lambda k: -len(m.acc[k].storage))  # 40, 3, 1 slots
    big, small, one = rich
    bare = next(k for k in keys if not m.acc[k].storage)
    ghost = b"\x05" * 32
    sk = sorted(m.acc[big].storage)
    ssz = [32 + len(slot_body(m.acc[big].storage[k])) for k in sk]
    tot_small = sum(32 + len(slot_body(v)) for v in m.acc[small].storage.values())
    sr = []
    for b in (0, 1, 32, 33, 34, 300, ssz[0], sum(ssz[:4]), sum(ssz[:4]) - 1, sum(ssz), sum(ssz) + 1, tot_small, tot_small + 1, 2 << 20, 1 << 63):
        sr.append(([big, small, one], ZERO, FF, b))                    # the first account cut
        sr.append(([small, big, one], ZERO, FF, b))                    # stop at a later account's first slot; budget at an end
        sr.append(([small, ghost, bare, one, big], ZERO, FF, b))       # absent and storage-less accounts in the middle
        sr.append(([big, small], sk[5], sk[9], b))                     # origin and limit on the first account only
        sr.append(([big, small], sk[5], add(sk[9], 1), b))
        sr.append(([big, big, small], add(sk[5], -1), sk[2], b))       # limit below origin; a repeated account
        sr.append(([big], add(sk[-1], 1), FF, b))                      # origin above every key
        sr.append(([small, big, one], ZERO, min(m.acc[small].storage), b))  # a limit with a zero origin: the later accounts whole
    return ar, sr


def test_cuts_and_bodies(lib, oracle):
    m = state(oracle)
    assert mismatches(lib, m, *cases(m)) == []


def test_random_states(lib, oracle):
    rng = np.random.default_rng(82)
    for t in range(4):
        d = Diff([(rng.bytes(32), 0, int(rng.integers(0, 1 << 20)), rng.bytes(int(rng.integers(0, 33))).rjust(32, b"\x00"),
                   EMPTY_CODE if rng.random() < 0.3 else rng.bytes(32)) for _ in range(int(rng.integers(1, 120)))])
        for i in range(0, len(d.accounts), 4):
            d.slots += [(i, rng.bytes(32), rng.bytes(int(rng.integers(1, 33))).rjust(32, b"\x00")) for _ in range(int(rng.integers(0, 30)))]
        m = StateModel(oracle)
        m.apply(Diff(d.accounts, [s for s in d.slots if s[2] != bytes(32)]))
        keys = sorted(m.acc)
        rich = [k for k in keys if m.acc[k].storage] or keys[:1]
        ar = [(add(keys[int(rng.integers(0, len(keys)))], int(rng.integers(-1, 2))), FF, int(rng.integers(0, 3000))) for _ in range(40)]
        sr = [([rich[int(i)] for i in rng.integers(0, len(rich), 5)], ZERO, FF, int(rng.integers(0, 3000))) for _ in range(40)]
        assert mismatches(lib, m, ar, sr) == [], t


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_mutants_fail(oracle, tmp_path, mutant):
    old, new = MUTANTS[mutant]
    text = open(os.path.join(CSRC, "snap_range.cuh")).read()
    assert text.count(old) == 1, mutant
    L = build(str(tmp_path), text.replace(old, new))
    m = state(oracle)
    assert mismatches(L, m, *cases(m)), mutant
