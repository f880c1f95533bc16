"""The device statements of the resident code store (phant_b200/csrc/resident_code.cuh) compiled as HOST code
(tests/hostcheck/resident_code_host.cpp) and held to the model of tests/resident_code_model.py across block sequences: put,
apply, revert, set_journal and prune.  Blocks go through tests/resident_state_model.py with each apply's undo record laid out as
the device lays it out (test_resident_read_header_host.record), except that a DELETE entry's code field -- zero on the device,
meaningless by the ABI -- holds the hash of a held decoy code that no account ever names, so that a store that counted DELETE
entries would keep it.  After every prune the kept set must be exactly the model's, which is stated on the reachable states
themselves, not on the records; at every `back` every account's code must look up as the model holds it, and every code that
was put, and not dropped while no reachable root named it, must be held while one does.  Two mutants of the header -- DELETE entries counted, records
ignored -- must each fail a case."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from resident_code_model import EMPTY_CODE_HASH, CodeStore
from resident_state_model import DELETE, ZERO32, Diff
from test_resident_read_header_host import RdRec, Reader, cat, record, rk, tables, val

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(ROOT, "phant_b200", "csrc")
RECORD_CODE = "return (R.aflags[p] & PHANT_GPU_ACCOUNT_DELETE) ? nullptr : R.code + 32ull * p;"
MUTANTS = {"delete entries counted": "return R.code + 32ull * p;", "records ignored": "return nullptr;"}


def build(out_dir, header=None):
    """the harness as a shared object; `header`: resident_code.cuh's text in place of the file's"""
    inc = [os.path.join(ROOT, "include"), CSRC]
    if header is not None:
        with open(os.path.join(out_dir, "resident_code.cuh"), "w") as f:
            f.write(header)
        inc.insert(0, str(out_dir))
    so = os.path.join(out_dir, "libresidentcodehost.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-Wno-unknown-pragmas", "-o", so] + [f"-I{d}" for d in inc] +
                   [os.path.join(HERE, "hostcheck", "resident_code_host.cpp")], check=True)
    L = C.CDLL(so)
    vp = C.c_void_p
    L.hc_lookup.argtypes = [vp, C.c_uint32, C.c_char_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint32)]
    L.hc_marks.argtypes = [vp, C.c_uint32, vp, vp, C.c_uint32, vp, C.c_uint32, vp]
    return L


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    return build(tmp_path_factory.mktemp("residentcodehost"))


def code_table(held):
    """a store as the device holds it: rows sorted by hash (key, arena offset, length) and the arena, 16-byte aligned"""
    hs = sorted(held)
    rows = np.zeros((max(len(hs), 1), 80), np.uint8)
    parts, off = [], 0
    for i, h in enumerate(hs):
        c = held[h]
        rows[i, :32] = np.frombuffer(h, np.uint8)
        rows[i, 32:40] = np.frombuffer(np.uint64(off).tobytes(), np.uint8)
        rows[i, 40:44] = np.frombuffer(np.uint32(len(c)).tobytes(), np.uint8)
        pad = -len(c) % 16
        parts.append(c + bytes(pad))
        off += len(c) + pad
    return hs, rows, cat(parts, 16)


class Coder(Reader):
    """Reader's block sequence with a journal depth, revert, and two stores: the model's and the one the header prunes"""

    def __init__(self, oracle, L, depth=1024):
        super().__init__(oracle)
        self.L, self.depth = L, depth
        self.keccak = oracle.keccak256
        self.model, self.dev = CodeStore(self.keccak), {}
        self.ever, self.bad = set(), []  # hashes of the non-empty codes put and not dropped by a model prune; mismatches
        self.decoy = self.put([b"\xfe decoy: held, never named " + bytes(8)])[0]

    def put(self, codes):
        hs = self.model.put(codes)
        for h, c in zip(hs, codes):
            if c:
                self.dev.setdefault(h, bytes(c))
                self.ever.add(h)
        return hs

    def apply(self, d):
        r, na, ms = record(self.m, d)
        for p in range(na):
            if r["aflags"][p] & DELETE:
                r["code"][32 * p:32 * p + 32] = np.frombuffer(self.decoy, np.uint8)
        self.journal.append((r, na, ms))
        self.m.apply(d)
        self.hist.append(self.m.copy())
        self.set_journal(self.depth)

    def revert(self, n):
        del self.journal[len(self.journal) - n:]
        del self.hist[len(self.hist) - n:]
        self.m = self.hist[-1].copy()

    def set_journal(self, depth):
        self.depth = depth
        if len(self.journal) > depth:
            del self.journal[:len(self.journal) - depth]

    def states(self):
        return [self.hist[len(self.hist) - 1 - b] for b in range(len(self.journal) + 1)]

    def window(self):
        back = len(self.journal)
        return back, (RdRec * max(back, 1))(*[RdRec(*[r[f].ctypes.data for f, _ in RdRec._fields_[:9]], na, ms) for r, na, ms in self.journal])

    def prune(self, tag):
        krows, nK, arena, _, _ = tables(self.m)
        back, recs = self.window()
        hs, rows, _ = code_table(self.dev)
        keep = np.zeros(max(len(hs), 1), np.uint8)
        if self.L.hc_marks(krows.ctypes.data, nK, arena.ctypes.data, recs, back, rows.ctypes.data, len(hs), keep.ctypes.data):
            self.bad.append((tag, "account body"))
        self.dev = {h: self.dev[h] for i, h in enumerate(hs) if keep[i]}
        self.model.prune(self.states())
        self.ever &= set(self.model.held)
        if set(self.dev) != set(self.model.held):
            self.bad.append((tag, "kept", sorted(h.hex()[:8] for h in set(self.dev) ^ set(self.model.held))))

    def check(self, tag, ghost_hashes=()):
        """every account's code at every back, and hashes nobody names"""
        hs, rows, arena = code_table(self.dev)
        off, ln = C.c_uint64(), C.c_uint32()
        for back, m in enumerate(self.states()):
            for k, a in m.acc.items():
                h = a.code_hash
                st = self.L.hc_lookup(rows.ctypes.data, len(hs), h, C.byref(off), C.byref(ln))
                got = (st == 1, arena[off.value:off.value + ln.value].tobytes() if st == 1 else b"")
                if got != self.model.lookup(h):
                    self.bad.append((tag, "lookup", back, k.hex()[:8]))
                if h in self.ever and st != 1:
                    self.bad.append((tag, "named code missing", back, k.hex()[:8]))
        for h in list(ghost_hashes) + [EMPTY_CODE_HASH]:
            st = self.L.hc_lookup(rows.ctypes.data, len(hs), h, C.byref(off), C.byref(ln))
            if (st == 1, ln.value if st == 1 else 0) != (self.model.lookup(h)[0], len(self.model.lookup(h)[1])):
                self.bad.append((tag, "ghost", h.hex()[:8]))


def account(k, code_hash, nonce=1):
    return (k, 0, nonce, (nonce * 7).to_bytes(32, "big"), code_hash)


def gone(k):
    return (k, DELETE, 0, ZERO32, ZERO32)


def code(rng, n=None):
    return rng.bytes(int(rng.integers(1, 300)) if n is None else n)


def scripted_recreate(r, rng):
    """a contract destroyed and re-created with different code across blocks, pruned in between"""
    a, b = rk(rng), rk(rng)
    c1, c2, c3 = code(rng), code(rng), code(rng, 1)
    h1, h2, h3 = r.put([c1, c2, c3])
    r.apply(Diff([account(a, h1), account(b, EMPTY_CODE_HASH)]))
    r.prune("created")
    r.apply(Diff([gone(a)]))
    r.apply(Diff())
    r.prune("destroyed")
    r.apply(Diff([account(a, h2)]))
    r.prune("re-created")
    r.apply(Diff([account(a, h3, 2), account(b, h2, 3)]))
    r.prune("changed")
    r.set_journal(1)
    r.prune("shallow")
    return [h1, h2, h3, rk(rng)]


def scripted_shared(r, rng):
    """one code shared by many accounts, one of them changed, then the rest one by one"""
    ks = [rk(rng) for _ in range(12)]
    s, t = code(rng, 700), code(rng, 64)
    hs, ht = r.put([s, t, s])[:2]
    r.apply(Diff([account(k, hs) for k in ks]))
    r.apply(Diff([account(ks[0], ht, 2)]))
    r.prune("one changed")
    r.set_journal(0)
    r.prune("no journal")
    for k in ks[1:]:
        r.apply(Diff([account(k, ht, 3)]))
    r.prune("all changed, journaled")
    r.set_journal(0)
    r.prune("all changed")
    return [hs, ht]


def scripted_record_only(r, rng):
    """a code named only by an undo record: kept while the record is in the window, dropped after"""
    x, y = rk(rng), rk(rng)
    old, new = code(rng), code(rng)
    ho, hn = r.put([old, new])
    r.apply(Diff([account(x, ho), account(y, ho)]))
    r.apply(Diff([account(x, hn, 2), gone(y)]))
    r.prune("named by the record only")
    r.apply(Diff())
    r.apply(Diff())
    r.prune("empty applies")
    r.revert(2)
    r.prune("reverted empties")
    r.set_journal(0)
    r.prune("record dropped")
    return [ho, hn]


def scripted_shallow(r, rng):
    """a deep journal, then a shallower one: the codes only the dropped records named go"""
    k = rk(rng)
    codes = [code(rng) for _ in range(8)]
    hs = r.put(codes)
    for i, h in enumerate(hs):
        r.apply(Diff([account(k, h, i + 1)]))
    r.prune("deep")
    r.set_journal(3)
    r.prune("shallow")
    r.revert(2)
    r.prune("reverted")
    r.set_journal(0)
    r.prune("none")
    return hs


def random_sequence(seed):
    def run(r, rng):
        keys = [rk(rng) for _ in range(10)]
        pool = r.put([code(rng) for _ in range(8)] + [b""])
        for step in range(16):
            x = rng.random()
            if x < 0.1:
                r.apply(Diff())
            elif x < 0.2 and r.journal:
                r.revert(int(rng.integers(1, len(r.journal) + 1)))
            elif x < 0.27:
                r.set_journal(int(rng.integers(0, 6)))
            elif x < 0.37:
                pool += r.put([code(rng) for _ in range(2)] + [r.model.held.get(pool[0], b"")])
            else:
                accounts, slots = [], []
                for k in rng.choice(len(keys), int(rng.integers(1, 5)), replace=False):
                    if rng.random() < 0.2:
                        accounts.append(gone(keys[k]))
                        continue
                    accounts.append(account(keys[k], pool[int(rng.integers(0, len(pool)))], int(rng.integers(1, 1 << 20))))
                    if rng.random() < 0.3:
                        slots.append((len(accounts) - 1, rk(rng), val(rng)))
                r.apply(Diff(accounts, slots))
            if rng.random() < 0.4:
                r.prune(f"step {step}")
            r.check(f"step {step}")
        r.prune("end")
        return pool
    return run


CASES = {"recreate": scripted_recreate, "shared": scripted_shared, "record only": scripted_record_only, "shallow": scripted_shallow} | \
    {f"random{i}": random_sequence(i) for i in range(6)}


def run_case(L, oracle, name):
    rng = np.random.default_rng(sorted(CASES).index(name) + 7)
    r = Coder(oracle, L, depth=int(rng.integers(4, 9)) if name.startswith("random") else 1024)
    ghosts = CASES[name](r, rng)
    r.check("end", ghosts + [rk(rng)])
    return r.bad


@pytest.mark.parametrize("case", sorted(CASES))
def test_store_across_blocks(lib, oracle, case):
    assert run_case(lib, oracle, case) == []


def test_record_only_code_is_kept(lib, oracle):
    """the code only a record names survives the first prune of that case and goes once the record leaves the window"""
    rng = np.random.default_rng(3)
    r = Coder(oracle, lib)
    ho, _ = scripted_record_only(r, rng)
    assert r.bad == [] and ho not in r.dev
    r2 = Coder(oracle, lib)
    x, y = rk(rng), rk(rng)
    ho, hn = r2.put([code(rng), code(rng)])
    r2.apply(Diff([account(x, ho), account(y, ho)]))
    r2.apply(Diff([account(x, hn, 2), gone(y)]))
    r2.prune("one record")
    assert r2.bad == [] and ho in r2.dev and r2.decoy not in r2.dev


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_mutants_fail(oracle, tmp_path, mutant):
    text = open(os.path.join(CSRC, "resident_code.cuh")).read()
    assert text.count(RECORD_CODE) == 1
    L = build(str(tmp_path), text.replace(RECORD_CODE, MUTANTS[mutant]))
    failed = [c for c in sorted(CASES) if run_case(L, oracle, c)]
    assert failed, mutant
