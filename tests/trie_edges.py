"""A seeded corpus of crafted tries whose nodes sit on the size edges of the trie encoders (phant_b200/csrc/trie.cu: the leaf,
branch and extension encoders, hdr_size / put_hdr / str_size, and the `len < 32` embedding rule), and a classifier that says
which edges the corpus really reaches.

Each case picks keys and values so that a named node lands on a named size: an RLP list or string payload on either side of
a header switch (55/56, 255/256, 65,535/65,536 bytes), a child of 31, 32 or 33 bytes (embedded or hashed) under a branch or an
extension, a branch value of those sizes, single-byte values (empty, 0x00, 0x7f, 0x80), and a one-key trie whose leaf is under
32 bytes (the root is hashed all the same).  Node sizes do not depend on the hash function (a hashed reference is always 33
bytes), so the cases are tuned with a stand-in hash and the classifier gives the same answer under Keccak.

classify(keccak, kv) re-parses every node helpers.py_mptize's recursion builds and returns one record per node;
labels(records) turns them into the edges reached.  TARGET_FLOORS holds, per edge, how many cases must reach it."""
import hashlib
from collections import Counter

import numpy as np

from helpers import _py_node, _rlp_item

BOUNDS = (55, 56, 255, 256, 65535, 65536)   # payload lengths on either side of each RLP header switch
CHILD_SIZES = (31, 32, 33)                  # a reference is the node itself below 32 bytes, its hash from 32 on
SINGLE = {b"": "empty", b"\x00": "0x00", b"\x7f": "0x7f", b"\x80": "0x80"}
KINDS = ("leaf at the root", "leaf under a branch", "extension", "branch without a value", "branch with a value")


def _stand_in(data):
    return hashlib.sha3_256(data).digest()


def _items(node):
    top = _rlp_item(node, 0, len(node))
    assert top is not None and top[0] and top[3] == len(node), node.hex()
    out, p = [], top[1]
    while p < top[2]:
        it = _rlp_item(node, p, top[2])
        assert it is not None
        out.append((it, node[p:it[3]]))
        p = it[3]
    return top[2] - top[1], out


def classify(keccak, kv):
    """every node of the trie over kv (sorted (key, value) pairs), root first: dicts with kind, size (bytes of the encoding),
    payload (bytes of the list payload), parent (None, "branch" or "extension"), value (leaf or branch value, else None) and
    path (hex-prefix bytes of a leaf or an extension, else None)"""
    seen = {}

    def h(data):
        d = keccak(data)
        seen[d] = data
        return d

    items = [([n for b in k for n in (b >> 4, b & 15)], v) for k, v in kv]
    root = _py_node(h, items, 0)
    recs = []

    def walk(node, parent):
        payload, its = _items(node)
        r = dict(size=len(node), payload=payload, parent=parent, value=None, path=None)
        recs.append(r)
        if len(its) == 2:
            (hp_it, _), (second, raw) = its
            hp = r["path"] = node[hp_it[1]:hp_it[2]]
            if hp[0] >> 4 & 2:
                r["kind"] = "leaf at the root" if parent is None else "leaf under a " + parent
                r["value"] = node[second[1]:second[2]]
            else:
                r["kind"] = "extension"
                child(second, raw, "extension")
        else:
            assert len(its) == 17
            val_it = its[16][0]
            r["value"] = node[val_it[1]:val_it[2]]
            r["kind"] = "branch with a value" if r["value"] else "branch without a value"
            for it, raw in its[:16]:
                if raw != b"\x80":
                    child(it, raw, "branch")

    def child(it, raw, parent):
        if it[0]:
            walk(raw, parent)                       # embedded: the node itself
        else:
            walk(seen[raw[1:]], parent)             # 0xa0 || digest

    walk(root, None)
    return recs


def labels(recs):
    """the edges a trie's node records reach (a Counter of label tuples)"""
    c = Counter()
    for r in recs:
        c[("kind", r["kind"])] += 1
        if r["payload"] in BOUNDS:
            c[("list payload", r["payload"])] += 1
        for s in (r["value"], r["path"]):
            if s is not None and len(s) in BOUNDS:
                c[("string payload", len(s))] += 1
        if r["parent"] and r["size"] in CHILD_SIZES:
            c[("child", r["parent"], r["size"])] += 1
        if r["kind"] == "branch with a value" and len(r["value"]) in CHILD_SIZES:
            c[("branch value", len(r["value"]))] += 1
        if r["value"] in SINGLE and r["kind"] != "branch without a value":  # a branch's empty value is no value
            c[("single-byte value", SINGLE[r["value"]])] += 1
        if r["parent"] is None and r["kind"] == "leaf at the root" and r["size"] < 32:
            c[("root", "leaf under 32 bytes")] += 1
    return c


# how many cases must reach each edge (a case counts once per edge, however many of its nodes reach it)
TARGET_FLOORS = {("kind", k): 5 for k in KINDS}
TARGET_FLOORS.update({("list payload", p): 3 for p in BOUNDS})
TARGET_FLOORS.update({("string payload", p): 2 for p in BOUNDS})
TARGET_FLOORS.update({("child", parent, s): 1 for parent in ("branch", "extension") for s in CHILD_SIZES})
TARGET_FLOORS.update({("branch value", s): 1 for s in CHILD_SIZES})
TARGET_FLOORS.update({("single-byte value", d): 2 for d in SINGLE.values()})
TARGET_FLOORS[("root", "leaf under 32 bytes")] = 1


class Case:
    def __init__(self, name, kv, targets):
        self.name, self.kv, self.targets = name, kv, list(targets)


def _tune(make, want, lo, hi):
    """the first p in [lo, hi) whose trie make(p) has a node record r with want(r)"""
    for p in range(lo, hi):
        kv = make(p)
        if any(want(r) for r in classify(_stand_in, kv)):
            return kv
    raise AssertionError("no parameter in range reaches the edge")


def _near(x, span=12):
    return max(0, x - span), x + span


def corpus(seed=2718):
    """the crafted cases, each with the edges it is built to reach"""
    rng = np.random.default_rng(seed)

    def val(n, first=None):
        v = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
        return v if first is None or not n else bytes([first]) + v[1:]

    big = val(40, 0xc4)  # a leaf value that makes its leaf hashed
    cases = [Case("one-key trie with a leaf under 32 bytes", [(b"\x01", b"\x02")],
                  [("kind", "leaf at the root"), ("root", "leaf under 32 bytes")])]

    # ---- single-byte and empty values: as the root leaf, as a leaf under a branch, as a branch value
    for v, d in SINGLE.items():
        cases.append(Case(f"root leaf value {d}", [(b"\xab", v)], [("single-byte value", d), ("kind", "leaf at the root")]))
        cases.append(Case(f"leaf value {d} under a branch", [(b"\x10", v), (b"\x20", big)],
                          [("single-byte value", d), ("kind", "leaf under a branch")]))
        if v:
            cases.append(Case(f"branch value {d}", [(b"\x01", v), (b"\x01\x20", big), (b"\x01\x30", b"z")],
                              [("single-byte value", d), ("kind", "branch with a value")]))
    # a key that is a prefix of another and holds the empty value: its branch encodes as one without a value
    cases.append(Case("prefix key with the empty value", [(b"\x01", b""), (b"\x01\x20", big), (b"\x01\x30", b"z")],
                      [("kind", "branch without a value"), ("kind", "extension")]))

    # ---- list and string headers on both sides of every switch
    for p in BOUNDS:
        cases.append(Case(f"root leaf, list payload {p}",
                          _tune(lambda x: [(b"\x5a", val(x, 0x91))], lambda r: r["parent"] is None and r["payload"] == p, *_near(p - 6)),
                          [("kind", "leaf at the root"), ("list payload", p)]))
        cases.append(Case(f"leaf under a branch, list payload {p}",
                          _tune(lambda x: [(b"\x10", val(x, 0x92)), (b"\x20", big)],
                                lambda r: r["kind"] == "leaf under a branch" and r["payload"] == p, *_near(p - 5)),
                          [("kind", "leaf under a branch"), ("list payload", p)]))
        cases.append(Case(f"branch with a value, list payload {p}",
                          _tune(lambda x: [(b"\x01", val(x, 0x93)), (b"\x01\x20", b"a"), (b"\x01\x30", b"b")],
                                lambda r: r["kind"] == "branch with a value" and r["payload"] == p, *_near(p - 24)),
                          [("kind", "branch with a value"), ("list payload", p)]))
        cases.append(Case(f"root leaf value, string payload {p}", [(b"\x33", val(p, 0x94))],
                          [("kind", "leaf at the root"), ("string payload", p)]))
        cases.append(Case(f"branch value, string payload {p}", [(b"\x01", val(p, 0x95)), (b"\x01\x20", big), (b"\x01\x30", b"c")],
                          [("kind", "branch with a value"), ("string payload", p)]))
    # a branch without a value: 55 / 56 with embedded children, 255 / 256 with hashed ones and one embedded child tuned
    for p in (55, 56):
        cases.append(Case(f"branch without a value, list payload {p}",
                          _tune(lambda x: [(b"\x10", val(x, 0x96)), (b"\x20", b"d" * 10), (b"\x30", b"e" * 10)],
                                lambda r: r["kind"] == "branch without a value" and r["payload"] == p, 1, 30),
                          [("kind", "branch without a value"), ("list payload", p)]))
    for p in (255, 256):
        cases.append(Case(f"branch without a value, list payload {p}",
                          _tune(lambda x: [(bytes([16 * j]), big) for j in range(7)] + [(b"\x70", val(x, 0x97))],
                                lambda r: r["kind"] == "branch without a value" and r["payload"] == p, 0, 40),
                          [("kind", "branch without a value"), ("list payload", p)]))
    # extensions: list payload 55 / 56 from the path length; a path string of 55 / 56 bytes (long-string header)
    for p in (55, 56):
        cases.append(Case(f"extension, list payload {p}",
                          _tune(lambda x: [(bytes(range(1, x + 1)) + b"\x10", big), (bytes(range(1, x + 1)) + b"\x20", big)],
                                lambda r: r["kind"] == "extension" and r["payload"] == p, 1, 40),
                          [("kind", "extension"), ("list payload", p)]))
        cases.append(Case(f"extension path string {p}",
                          _tune(lambda x: (lambda pre: [(pre + b"\x10", b"f"), (pre + b"\x20", b"g")])(val(x, 0x21)),
                                lambda r: r["kind"] == "extension" and len(r["path"]) == p, 50, 60),
                          [("kind", "extension"), ("string payload", p)]))
        cases.append(Case(f"leaf path string {p}", [(b"\x01" * (p - 1), b"h")], [("kind", "leaf at the root"), ("string payload", p)]))

    # ---- children of 31 / 32 / 33 bytes under a branch (leaf, branch and extension children) and under an extension
    for s in CHILD_SIZES:
        cases.append(Case(f"leaf child of {s} bytes under a branch",
                          _tune(lambda x: [(b"\x10", val(x, 0x98)), (b"\x20", big)],
                                lambda r: r["kind"] == "leaf under a branch" and r["size"] == s, 20, 40),
                          [("child", "branch", s)]))
        cases.append(Case(f"branch child of {s} bytes under a branch",
                          _tune(lambda x: [(b"\x10", val(x, 0x99)), (b"\x11", b"i"), (b"\x20", big)],
                                lambda r: r["parent"] == "branch" and r["kind"].startswith("branch") and r["size"] == s, 1, 30),
                          [("child", "branch", s), ("kind", "branch without a value")]))
        cases.append(Case(f"extension child of {s} bytes under a branch",
                          _tune(lambda x: [(b"\x10\x01", val(x, 0x9a)), (b"\x10\x02", b"j"), (b"\x20", big)],
                                lambda r: r["kind"] == "extension" and r["parent"] == "branch" and r["size"] == s, 1, 30),
                          [("child", "branch", s), ("kind", "extension")]))
        cases.append(Case(f"branch child of {s} bytes under an extension",
                          _tune(lambda x: [(b"\xab\x10", val(x, 0x9b)), (b"\xab\x20", b"k")],
                                lambda r: r["parent"] == "extension" and r["size"] == s, 1, 30),
                          [("child", "extension", s), ("kind", "extension")]))
        cases.append(Case(f"branch value of {s} bytes", [(b"\x01", val(s, 0x9c)), (b"\x01\x20", b"l"), (b"\x01\x30", big)],
                          [("branch value", s), ("kind", "branch with a value")]))
    return cases


def reached(keccak, cases):
    """Counter over the edges: how many cases reach each one"""
    c = Counter()
    for case in cases:
        c.update(set(labels(classify(keccak, case.kv))))
    return c
