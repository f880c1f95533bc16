"""The range-proof check (phant_gpu_verify_ranges, DESIGN.md §4.3j) stated on the CPU for the tests, written from the header's
statement with go-ethereum's method (VerifyRangeProof), not the GPU's: build a partial trie from the boundary proofs' nodes,
remove every reference strictly between the two edge paths, insert the entries, hash and compare with the root; `more` is
whether anything is left to the right of the last key's path.  Removing references can leave a branch with one child: it
collapses as a trie delete would, resolving that child when the branch references it by hash (a child below an extension is
a branch, known without a lookup).  TEST INFRASTRUCTURE: the product never imports this."""
from helpers import _hp, rlp_list, rlp_str
from transition_oracle import BAD, EMPTY_ROOT, MISSING, decode, nibbles, status_of

WHOLE = 1
FF32 = b"\xff" * 32

# partial-trie nodes: None (empty), ("hash", digest, below_ext) (not resolved), ("raw", node bytes) (an embedded node kept as it
# is), ("leaf", path, value), ("ext", path, child), ("branch", [16 children]); paths are tuples of nibbles


def entries_ok(entries, origin, whole):
    """strictly ascending keys, none below the origin (unless WHOLE), no empty value"""
    for i, (k, v) in enumerate(entries):
        if not v or (i and entries[i - 1][0] >= k) or (not whole and k < origin):
            return False
    return True


def last_key(entries):
    return entries[-1][0] if entries else FF32


class _Check:
    def __init__(self, keccak, table):
        self.kc, self.table, self.flags, self.more = keccak, table, 0, False

    # ---- the partial trie: the nodes on the edge paths, and every embedded node ----
    def resolve(self, ref, node, prefix, edges, below_ext=False):
        if node is None:
            if not any(e[:len(prefix)] == prefix for e in edges):
                return ("hash", ref, below_ext)
            node = self.table.get(ref)
            if node is None:
                self.flags |= MISSING
                return None
        t = decode(node)
        d = len(prefix)
        if t is None:
            self.flags |= BAD
            return None
        if t[0] == "leaf":
            if d + len(t[1]) != 64:
                self.flags |= BAD
                return None
            return ("leaf", t[1], t[2])
        if t[0] == "ext":
            if d + len(t[1]) >= 64:
                self.flags |= BAD
                return None
            return ("ext", t[1], self.child(t[2], prefix + t[1], edges, True))
        if d >= 64:
            self.flags |= BAD
            return None
        return ("branch", [None if c is None else self.child(c, prefix + (v,), edges, False) for v, c in enumerate(t[1])])

    def child(self, c, prefix, edges, below_ext):
        return self.resolve(c[1], None, prefix, edges, below_ext) if c[0] == "hash" else self.resolve(None, c[1], prefix, edges)

    # ---- remove every reference strictly between the edge paths ----
    def unset(self, node, prefix, lo, hi):
        """drop each leaf in [lo, hi] and each unresolved subtree whose prefix interval lies inside it; note what stays above hi"""
        if node is None:
            return None
        if node[0] in ("hash", "leaf"):
            key = prefix + (node[1] if node[0] == "leaf" else ())
            first, end = key + (0,) * (64 - len(key)), key + (15,) * (64 - len(key))
            if lo <= first and end <= hi:
                return None
            self.more |= first > hi
            return node
        if node[0] == "ext":
            c = self.unset(node[2], prefix + node[1], lo, hi)
            return None if c is None else ("ext", node[1], c)
        return ("branch", [self.unset(c, prefix + (v,), lo, hi) for v, c in enumerate(node[1])])

    # ---- insert the entries ----
    def insert(self, node, rest, value):
        if node is None:
            return ("leaf", rest, value)
        kind = node[0]
        if kind == "branch":
            kids = list(node[1])
            kids[rest[0]] = self.insert(kids[rest[0]], rest[1:], value)
            return ("branch", kids)
        assert kind in ("leaf", "ext"), kind  # an unresolved subtree lies outside the range, and so does every key under it
        path = node[1]
        if kind == "leaf" and path == rest:
            return ("leaf", rest, value)
        if kind == "ext" and rest[:len(path)] == path:
            return ("ext", path, self.insert(node[2], rest[len(path):], value))
        c = 0
        while path[c] == rest[c]:
            c += 1
        kids = [None] * 16
        tail = path[c + 1:]
        if kind == "leaf":
            kids[path[c]] = ("leaf", tail, node[2])
        else:
            kids[path[c]] = ("ext", tail, node[2]) if tail else node[2]
        kids[rest[c]] = ("leaf", rest[c + 1:], value)
        br = ("branch", kids)
        return ("ext", path[:c], br) if c else br

    # ---- collapse what the removal left with fewer than two children ----
    def collapse(self, node, depth):
        if node is None or node[0] in ("hash", "leaf", "raw"):
            return node
        if node[0] == "ext":
            c = self.collapse(node[2], depth + len(node[1]))
            if c is None:
                return None
            if c[0] == "leaf":
                return ("leaf", node[1] + c[1], c[2])
            if c[0] == "ext":
                return ("ext", node[1] + c[1], c[2])
            return ("ext", node[1], c)
        kids = [self.collapse(c, depth + 1) for c in node[1]]
        live = [v for v in range(16) if kids[v] is not None]
        if not live:
            return None
        if len(live) > 1:
            return ("branch", kids)
        v = live[0]
        c = kids[v]
        if c[0] == "hash" and not c[2]:
            c = self.lookup_moved(c[1], depth + 1)
            if c is None:
                return ("branch", kids)  # the status is already decided
        if c[0] == "leaf":
            return ("leaf", (v,) + c[1], c[2])
        if c[0] == "ext":
            return ("ext", (v,) + c[1], c[2])
        return ("ext", (v,), c)

    def lookup_moved(self, ref, depth):
        """the node an unresolved child becomes when its parent branch goes: a leaf, an extension, or a branch kept by hash"""
        node = self.table.get(ref)
        if node is None:
            self.flags |= MISSING
            return None
        t = decode(node)
        if t is None or (t[0] == "leaf" and depth + len(t[1]) != 64) or (t[0] == "ext" and depth + len(t[1]) >= 64):
            self.flags |= BAD
            return None
        if t[0] == "leaf":
            return ("leaf", t[1], t[2])
        if t[0] == "ext":
            return ("ext", t[1], ("hash", t[2][1], True) if t[2][0] == "hash" else ("raw", t[2][1]))
        return ("hash", ref, True)

    # ---- hash ----
    def encode(self, node):
        kind = node[0]
        if kind == "leaf":
            return rlp_list([rlp_str(_hp(node[1], True)), rlp_str(node[2])])
        if kind == "ext":
            return rlp_list([rlp_str(_hp(node[1], False)), self.ref(node[2])])
        return rlp_list([rlp_str(b"") if c is None else self.ref(c) for c in node[1]] + [rlp_str(b"")])

    def ref(self, node):
        if node[0] == "hash":
            return rlp_str(node[1])
        if node[0] == "raw":
            return node[1]
        enc = self.encode(node)
        return enc if len(enc) < 32 else rlp_str(self.kc(enc))

    def root(self, node):
        return EMPTY_ROOT if node is None else node[1] if node[0] == "hash" else self.kc(self.encode(node))


def verify_range(keccak, nodes, root, origin, entries, whole=False):
    """one range: entries [(key32, value)] under `root` -> (status 1 / 0 / 3, more); nodes: the node set, a list of node
    bytes or {digest: node} (many ranges over one set)"""
    if not entries_ok(entries, origin, whole):
        return 0, False
    chk = _Check(keccak, nodes if isinstance(nodes, dict) else {keccak(n): n for n in nodes})
    lo, hi = nibbles(origin), nibbles(last_key(entries))
    trie = None
    if not whole and root != EMPTY_ROOT:
        trie = chk.resolve(root, None, (), (lo, hi))
        if chk.flags:
            return status_of(chk.flags), False
        trie = chk.unset(trie, (), lo, hi)
    for k, v in entries:
        trie = chk.insert(trie, nibbles(k), v)
    trie = chk.collapse(trie, 0)
    if chk.flags:
        return status_of(chk.flags), False
    if chk.root(trie) != root:
        return 0, False
    return 1, chk.more
