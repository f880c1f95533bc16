"""The device range statements of the resident world state (phant_b200/csrc/resident_range.cuh) compiled as HOST code and
run as one whole range call (tests/hostcheck/resident_range_host.cpp: parts, candidates, sort, dedupe, resolution, ranks,
selection, fill), held to the Python model at every root a journal reaches.  Block sequences and undo records are those
of test_resident_read_header_host.py (the device's layout).  Every range at every `back` must equal the model's snapshot of
that block, `more` and storage roots included, and each range's candidates must stay within entries + 1 + 2R (R: the
window's record keys inside the range), the device-memory bound the call promises.  Two mutants of the header -- the
candidate bound max + R in place of max + 1 + R, and no DELETE / CLEAR_STORAGE exception -- must each fail a case."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from resident_range_model import MAX_KEY, ZERO_KEY, add, expect, ranges_over
from resident_state_model import CLEAR, DELETE, ZERO32, Diff
from resident_state_undo import snapshot
from test_resident_read_header_host import RdRec, Reader, rk, tables, val

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "phant_b200", "csrc")
MUTANTS = {"max+R": ("const uint64_t want = (uint64_t)max + 1 + R;", "const uint64_t want = (uint64_t)max + R;", 2),
           "no exception": ("now = false;", "(void)now;", 1)}


def build(out_dir, header=None):
    """the harness as a shared object; `header`: resident_range.cuh's text in place of the file's"""
    inc = [os.path.join(ROOT, "include"), CSRC]
    if header is not None:
        with open(os.path.join(out_dir, "resident_range.cuh"), "w") as f:
            f.write(header)
        inc.insert(0, str(out_dir))
    so = os.path.join(out_dir, "libresidentrangehost.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so] + [f"-I{d}" for d in inc] +
                   [os.path.join(HERE, "hostcheck", "resident_range_host.cpp")], check=True)
    L = C.CDLL(so)
    vp = C.c_void_p
    L.hr_range.argtypes = [vp, C.c_uint32, vp, vp, C.c_uint32, vp, C.c_uint32, C.c_uint32, C.c_uint32, vp, vp, vp, vp, C.c_uint64,
                           vp, vp, vp, vp, vp, vp, vp]
    return L


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return build(tmp_path_factory.mktemp("residentrangehost"))


def listed(rec):
    """an undo record's account keys and, per listed account, its listed slot keys"""
    r, na, ms = rec
    ak = [r["akeys"][32 * i:32 * i + 32].tobytes() for i in range(na)]
    slots = {}
    for j in range(ms):
        slots.setdefault(ak[int(r["sacc"][j])], []).append(r["skeys"][32 * j:32 * j + 32].tobytes())
    return ak, slots


class Ranger(Reader):
    def run(self, L, aranges, sranges):
        """every range at every back; returns the mismatches (empty: all equal the model)"""
        krows, n, arena, srows, nS = tables(self.m)
        bad = []
        cat = lambda xs: np.frombuffer(b"".join(xs) or bytes(32), np.uint8).copy()  # noqa: E731
        na, ms = len(aranges), len(sranges)
        origin, limit = cat([r[0] for r in aranges] + [r[1] for r in sranges]), cat([r[1] for r in aranges] + [r[2] for r in sranges])
        sacct = cat([r[0] for r in sranges])
        mx = np.array([r[2] for r in aranges] + [r[3] for r in sranges] + [0], np.uint32)
        for back in range(len(self.journal) + 1):
            win = self.journal[len(self.journal) - back:]
            recs = (RdRec * max(back, 1))(*[RdRec(*[r[f].ctypes.data for f, _ in RdRec._fields_[:9]], a, s) for r, a, s in win])
            h = self.hist[len(self.hist) - 1 - back]
            snap = snapshot(h)
            keys = sorted(snap)
            cap = sum(min(int(x), len(keys) + 64) for x in mx[:na]) + sum(min(int(x), 4096) for x in mx[na:na + ms]) + 1
            first, more, cands = np.zeros(na + ms + 1, np.uint64), np.zeros(na + ms + 1, np.uint8), np.zeros(na + ms + 1, np.uint64)
            ek, nonce, acc, sv = np.zeros((cap, 32), np.uint8), np.zeros(cap, np.uint64), np.zeros((cap, 96), np.uint8), np.zeros((cap, 32), np.uint8)
            rc = L.hr_range(krows.ctypes.data, n, arena.ctypes.data, srows.ctypes.data, nS, recs, back, na, ms, origin.ctypes.data,
                            limit.ctypes.data, sacct.ctypes.data, mx.ctypes.data, cap, first.ctypes.data, more.ctypes.data,
                            cands.ctypes.data, ek.ctypes.data, nonce.ctypes.data, acc.ctypes.data, sv.ctypes.data)
            if rc:
                bad.append((back, "rc", rc))
                continue
            lists = [listed(r) for r in win]
            for r, (o, lim, m) in enumerate(aranges):
                want, want_more = expect(keys, o, lim, m)
                e = range(int(first[r]), int(first[r + 1]))
                got = [ek[i].tobytes() for i in e]
                if got != want or bool(more[r]) != want_more:
                    bad.append((back, "account range", r))
                    continue
                for i, k in zip(e, got):
                    nn, bal, ch, _ = snap[k]
                    if (int(nonce[i]), acc[i, :32].tobytes(), acc[i, 32:64].tobytes(), acc[i, 64:].tobytes()) != (nn, bal, h.storage_root(k), ch):
                        bad.append((back, "account value", r, k.hex()))
                R = sum(sum(o <= k <= lim for k in ak) for ak, _ in lists)
                if int(cands[r]) > len(want) + 1 + 2 * R:
                    bad.append((back, "account candidates", r, int(cands[r]), len(want), R))
            for s, (ak, o, lim, m) in enumerate(sranges):
                r = na + s
                st = {k: v for k, v in snap[ak][3].items() if v != ZERO32} if ak in snap else {}
                want, want_more = expect(sorted(st), o, lim, m)
                e = range(int(first[r]), int(first[r + 1]))
                got = [ek[i].tobytes() for i in e]
                if got != want or bool(more[r]) != want_more:
                    bad.append((back, "storage range", s))
                    continue
                if any(sv[i].tobytes() != st[k] for i, k in zip(e, got)):
                    bad.append((back, "slot value", s))
                R = sum(sum(o <= k <= lim for k in sl.get(ak, ())) for _, sl in lists)
                if int(cands[r]) > len(want) + 1 + 2 * R:
                    bad.append((back, "storage candidates", s, int(cands[r]), len(want), R))
        return bad


def storage_ranges(r, rng, accounts, n):
    """n storage ranges per account over every slot key the account ever held"""
    out = []
    for a in accounts:
        sks = sorted({sk for h in r.hist if a in h.acc for sk in h.acc[a].storage})
        out += [(a,) + x for x in ranges_over(sks, rng, n)]
    return out


def scripted(seed=1):
    """1,000 accounts inserted at the front of a range; an account destroyed and re-created across the window;
    CLEAR_STORAGE then newer writes; a slot-rich account re-created with more slots than it had; empty applies"""
    def run(oracle):
        rng = np.random.default_rng(seed)
        r = Ranger(oracle)
        hi = [b"\x80" + rk(rng)[1:] for _ in range(40)]
        lo_keys = [b"\x10" + rk(rng)[1:] for _ in range(1000)]
        a, b, c = hi[0], hi[1], hi[2]
        s = [b"\x40" + rk(rng)[1:] for _ in range(8)]
        many = [b"\x41" + rk(rng)[1:] for _ in range(300)]
        f = lambda n: (n, (n * 7).to_bytes(32, "big"), rk(rng))  # noqa: E731
        r.apply(Diff([(k, 0) + f(i + 1) for i, k in enumerate(hi)], [(0, k, val(rng)) for k in s[:4]] + [(1, k, val(rng)) for k in s]))
        r.apply(Diff())                                                                        # empty
        r.apply(Diff([(k, 0) + f(5) for k in lo_keys]))                                        # 1,000 in front
        r.apply(Diff([(a, DELETE, 0, ZERO32, ZERO32)]))                                        # destroy
        r.apply(Diff([(a, 0) + f(3)], [(0, s[5], val(rng))]))                                  # re-create
        r.apply(Diff([(b, CLEAR) + f(4)], [(0, s[6], val(rng))] + [(0, k, val(rng)) for k in many]))  # clear, many writes
        r.apply(Diff([(b, 0) + f(6)], [(0, s[2], val(rng)), (0, s[7], val(rng)), (0, s[6], ZERO32)]))  # newer writes
        r.apply(Diff([(c, 0) + f(7)], [(0, s[0], val(rng))]))
        r.apply(Diff())
        keys = sorted({k for h in r.hist for k in h.acc}) + [b"\x90" + rk(rng)[1:]]
        ar = ranges_over(keys[:20] + keys[-30:], rng, 120) + [(ZERO_KEY, MAX_KEY, 10), (lo_keys[0], MAX_KEY, 10), (add(max(lo_keys), 1), MAX_KEY, 1)]
        sr = storage_ranges(r, rng, [a, b, c, hi[3], keys[-1]], 40)
        return r, ar, sr
    return run


def random_sequence(seed):
    def run(oracle):
        rng = np.random.default_rng(100 + seed)
        r = Ranger(oracle)
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
        return r, ranges_over(keys, rng, 60), storage_ranges(r, rng, keys + [rk(rng)], 12)
    return run


CASES = {"scripted": scripted()} | {f"random{i}": random_sequence(i) for i in range(6)}


@pytest.mark.parametrize("case", sorted(CASES))
def test_ranges_at_every_back(lib, oracle, case):
    r, ar, sr = CASES[case](oracle)
    assert r.run(lib, ar, sr) == []


def test_front_insert_is_skipped(lib, oracle):
    """the 1,000 accounts the third block put in front: one back before it, a max-10 range from 0 skips every one"""
    r, _, _ = CASES["scripted"](oracle)
    before = r.hist[2]
    assert len(r.hist[3].acc) - len(before.acc) == 1000
    assert r.run(lib, [(ZERO_KEY, MAX_KEY, 10), (ZERO_KEY, MAX_KEY, 0), (MAX_KEY, ZERO_KEY, 5)], []) == []


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_mutants_fail(oracle, tmp_path, mutant):
    """each mutant of the header breaks at least one case: the max + R bound misses `more` where R current keys drop out,
    and without the exception the candidates of a cleared account outgrow entries + 1 + 2R"""
    old, new, count = MUTANTS[mutant]
    text = open(os.path.join(CSRC, "resident_range.cuh")).read()
    assert text.count(old) == count, mutant
    L = build(str(tmp_path), text.replace(old, new))
    failed = []
    for c in sorted(CASES):
        r, ar, sr = CASES[c](oracle)
        if r.run(L, ar, sr):
            failed.append(c)
    assert failed, mutant
