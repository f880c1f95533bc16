"""Range-proof answers with known truth, shared by the CPU statement's tests, the host-compiled header's tests and the GPU tests:
tries whose contents are known (every account and storage trie of the fixture states, random tries, tries with awkward
shapes), answers served from them the way a snap server serves them (entries from an origin, the proofs of the origin and of
the last entry), and mutations of those answers that must never be accepted.  TEST INFRASTRUCTURE."""
import bisect

import numpy as np

from helpers import rlp_str
from resident_state_model import StateModel, hashed_table, load_diff
from transition_oracle import EMPTY_ROOT

FF32 = b"\xff" * 32


def key_after(k):
    return (int.from_bytes(k, "big") + 1).to_bytes(32, "big")


def key_before(k):
    return (int.from_bytes(k, "big") - 1).to_bytes(32, "big")


class KnownTrie:
    """sorted [(key32, value)] and the oracle's trie over them"""

    def __init__(self, oracle, kv, name=""):
        self.kv, self.name = sorted(kv), name
        self.keys = [k for k, _ in self.kv]
        self.trie = oracle.trie(self.kv) if self.kv else None
        self.root = self.trie.root() if self.kv else EMPTY_ROOT

    def prove(self, key):
        return self.trie.prove(key) if self.trie else []

    def serve(self, origin, count):
        """(entries, proof nodes, more): up to `count` entries from `origin`, with the proofs of the origin and the last entry"""
        i = bisect.bisect_left(self.keys, origin)
        ents = self.kv[i:i + count]
        nodes = dict.fromkeys(self.prove(origin))
        if ents:
            nodes.update(dict.fromkeys(self.prove(ents[-1][0])))
        return ents, list(nodes), i + len(ents) < len(self.kv)

    def origins(self, limit=None, rng=None):
        """every key, a key between each pair of neighbours, one below the first key and one above the last"""
        out = {bytes(32), FF32}
        for i, k in enumerate(self.keys):
            out.add(k)
            if k != FF32 and (i + 1 == len(self.keys) or key_after(k) != self.keys[i + 1]):
                out.add(key_after(k))
            if k != bytes(32):
                out.add(key_before(k))
        out = sorted(out)
        if limit and len(out) > limit:
            out = [out[int(j)] for j in sorted(rng.choice(len(out), limit, replace=False))]
        return out


def fixture_tries(oracle, golden):
    """every account trie and every storage trie of the fixture states' tables"""
    g = golden("fixture_states.json.gz")
    out = []
    for name, table in g["tables"].items():
        m = StateModel(oracle)
        m.apply(load_diff(hashed_table(oracle.keccak256, table)))
        out.append(KnownTrie(oracle, [(k, m.leaf(k)) for k in m.acc], f"{name}/accounts"))
        for k, a in m.acc.items():
            live = {sk: v for sk, v in a.storage.items() if v != bytes(32)}
            if live:
                out.append(KnownTrie(oracle, [(sk, rlp_str(v.lstrip(b"\x00"))) for sk, v in live.items()], f"{name}/{k.hex()[:8]}"))
    return out


def random_tries(oracle, seed=7):
    rng = np.random.default_rng(seed)
    out = []
    for n, vlen in ((40, 70), (200, 3), (600, 40)):
        kv = {bytes(rng.integers(0, 256, 32, dtype=np.uint8)): bytes(rng.integers(1, 256, vlen, dtype=np.uint8)) for _ in range(n)}
        out.append(KnownTrie(oracle, list(kv.items()), f"random{n}"))
    return out


def awkward_tries(oracle, seed=11):
    """keys sharing 62 or more nibbles with short values (embedded leaves and subtrees), clusters under one extension, a
    single key, the empty trie"""
    rng = np.random.default_rng(seed)
    out = [KnownTrie(oracle, [], "empty"), KnownTrie(oracle, [(bytes(rng.integers(0, 256, 32, dtype=np.uint8)), b"\x01")], "single")]
    base = bytes(rng.integers(0, 256, 32, dtype=np.uint8))
    emb = {base[:31] + bytes([b]): bytes([1 + i % 100]) for i, b in enumerate((0x00, 0x01, 0x07, 0x10, 0x11, 0x3f, 0xf0, 0xfe))}
    emb.update({bytes(rng.integers(0, 256, 32, dtype=np.uint8)): b"\x05" for _ in range(6)})
    out.append(KnownTrie(oracle, list(emb.items()), "embedded"))
    only = {base[:31] + bytes([b]): bytes([2 + b % 50]) for b in (0x20, 0x21, 0x2f)}
    out.append(KnownTrie(oracle, list(only.items()), "embedded-only"))
    ext = {}
    for c in range(5):  # five clusters, each under a long extension, each cluster's keys sharing 60 nibbles
        head = bytes(rng.integers(0, 256, 30, dtype=np.uint8))
        for j in range(4):
            ext[head + bytes([0x40 + j, 0x11 * j])] = bytes(rng.integers(1, 256, 40, dtype=np.uint8))
    out.append(KnownTrie(oracle, list(ext.items()), "extensions"))
    two = {bytes(31) + b"\x01": b"\x01" * 40, FF32[:31] + b"\xfe": b"\x02" * 40}
    out.append(KnownTrie(oracle, list(two.items()), "two"))
    return out


def accept_cases(t, counts=(1, 2, 3, None), limit=None, rng=None):
    """(origin, entries, nodes, whole, more) that a correct check accepts: each origin with each count (None: everything from
    it), the WHOLE answer, and an empty answer past the last key"""
    out = []
    for o in t.origins(limit, rng):
        for c in counts:
            ents, nodes, more = t.serve(o, len(t.kv) if c is None else c)
            out.append((o, ents, nodes, False, more))
    out.append((bytes(32), list(t.kv), [], True, False))
    if t.kv and t.keys[-1] != FF32:
        _, nodes, _ = t.serve(key_after(t.keys[-1]), 1)
        out.append((key_after(t.keys[-1]), [], nodes, False, False))
    return out


def truth(t, origin, entries, whole):
    """(whether the answer is exactly the trie's contents in [origin, last] -- all of them with WHOLE --, more)"""
    if whole:
        return list(entries) == t.kv, False
    last = entries[-1][0] if entries else FF32
    inside = [(k, v) for k, v in t.kv if origin <= k <= last]
    return list(entries) == inside, any(k > last for k in t.keys)


def mutations(t, origin, count, rng):
    """(name, root, origin, entries, nodes, whole) answers made from an honest answer of at least three entries that leaves
    a key after it.  Every one is a lie or a broken proof, except drop-last: without its last entry an answer is a shorter
    honest answer, which a check may accept when the proof holds the new last key's path (and must then report more)."""
    ents, nodes, _ = t.serve(origin, count)
    assert len(ents) >= 3
    root = t.root
    out = []
    mid = len(ents) // 2
    out.append(("drop-first", root, origin, ents[1:], nodes, False))
    out.append(("drop-middle", root, origin, ents[:mid] + ents[mid + 1:], nodes, False))
    out.append(("drop-last", root, origin, ents[:-1], nodes, False))
    lo, hi = int.from_bytes(ents[0][0], "big"), int.from_bytes(ents[-1][0], "big")
    have = set(t.keys)
    for _ in range(50):
        kb = (lo + 1 + int(rng.integers(0, 1 << 62)) % (hi - lo - 1)).to_bytes(32, "big") if hi - lo > 1 else None
        if kb is not None and kb not in have:
            out.append(("add-inside", root, origin, sorted(ents + [(kb, b"\x01")]), nodes, False))
            break
    v = bytearray(ents[mid][1])
    v[len(v) // 2] ^= 1
    out.append(("value-byte", root, origin, ents[:mid] + [(ents[mid][0], bytes(v))] + ents[mid + 1:], nodes, False))
    out.append(("swap", root, origin, ents[:mid - 1] + [ents[mid], ents[mid - 1]] + ents[mid + 1:], nodes, False))
    out.append(("duplicate", root, origin, ents[:mid] + [ents[mid]] + ents[mid:], nodes, False))
    out.append(("below-origin", root, key_after(ents[0][0]), ents, nodes, False))
    out.append(("empty-value", root, origin, ents[:mid] + [(ents[mid][0], b"")] + ents[mid + 1:], nodes, False))
    out.append(("empty-answer", root, origin, [], nodes, False))
    out.append(("whole-truncated", root, origin, ents, [], True))
    for j in range(len(nodes)):
        out.append((f"drop-node{j}", root, origin, ents, nodes[:j] + nodes[j + 1:], False))
        b = bytearray(nodes[j])
        b[len(b) // 2] ^= 0x10
        out.append((f"node-byte{j}", root, origin, ents, nodes[:j] + [bytes(b)] + nodes[j + 1:], False))
    for other in (bytes(32), FF32, t.keys[0], t.keys[-1]):
        onodes = list(dict.fromkeys(t.serve(other, 1)[1] + t.serve(ents[-1][0], 1)[1]))
        if not set(t.prove(origin)) <= set(onodes):
            out.append(("other-origin-proof", root, origin, ents, onodes, False))
            break
    out.append(("wrong-root", bytes(31) + b"\x01", origin, ents, nodes, False))
    return out


def mutation_cases(t, rng):
    """the mutations of two answers of t (from its second key, and from just after it), when t is large enough"""
    if len(t.kv) < 6:
        return []
    return mutations(t, t.keys[1], 4, rng) + mutations(t, key_after(t.keys[1]), 3, rng)
