"""A deterministic corpus of malformed proofs whose hashes still match, for the proof walk's decoding rules (R2-R4 of
DESIGN.md "Proof walk").

Damaging a node's bytes without touching its parent's reference only ever exercises R1: the hash check fails before any
decoding runs.  Every case here is linked: keccak(nodes[0]) is the root and each node down to the malformed one is named by
its parent (hash reference, or embedded in place), so the walk really reaches the malformed node and decides by R2-R4.

A case is built in three layers:
  - a *core* builds the node under test (plus any node its reference leads to) for the key nibbles left at its position,
    and states the status the rules prescribe, for the node as the chain's last node and as a node that is not last;
  - a *placement* puts it at depth 0, 1 or 5 (branches, and an extension to reach a given key position), last or not, or
    embedded in its parent where it is short enough;
  - `wrap` writes the ancestors over it, so their references and the root match.
`reseal` does the same for a node of a genuine proof: the random-damage cases apply test_fuzz_walk.damage to one node and
reseal its ancestors.

Pure Python plus the oracle's keccak; no GPU.  Used by test_walk_rules_corpus.py (host-compiled device sources) and
test_gpu_walk_rules_corpus.py (every device path)."""
import numpy as np

from helpers import EMPTY_ROOT, _hp, rlp_list, rlp_str

REJECT, PRESENT, ABSENT, MISSING = 0, 1, 2, 3


class Case:
    __slots__ = ("name", "nodes", "key", "root", "status", "value", "target")

    def __init__(self, name, nodes, key, root, status, value, target):
        self.name, self.nodes, self.key, self.root = name, nodes, key, root
        self.status, self.value = status, value  # prescribed; None for the random-damage cases (the oracle decides)
        self.target = target  # chain index of the node under test (None: it is embedded in its parent)

    def proof(self):
        return (self.nodes, self.key, self.root)


def key_bytes(nibs):
    assert len(nibs) == 64
    return bytes((nibs[2 * i] << 4) | nibs[2 * i + 1] for i in range(32))


def hashref(keccak, node):
    return rlp_str(keccak(node))


def leaf(path, value):
    return rlp_list([rlp_str(_hp(path, True)), rlp_str(value)])


def ext(path, child_item):
    return rlp_list([rlp_str(_hp(path, False)), child_item])


def long_list(payload, n_len=None):
    """a list header in long form whatever the payload's size; n_len length bytes (leading zeros) if given"""
    n = len(payload)
    lb = n.to_bytes(max(1, (n.bit_length() + 7) // 8), "big")
    if n_len is not None:
        lb = lb.rjust(n_len, b"\x00")
    return bytes([0xf7 + len(lb)]) + lb + payload


def payload_of(node):
    """the payload of a well-formed list node"""
    b = node[0]
    if b <= 0xf7:
        return node[1:]
    return node[1 + b - 0xf7:]


def reseal(keccak, chain, j, new_node):
    """replace node j of a hash-linked chain (every node after the root is named by a 32-byte hash in the node before it)
    and give each ancestor the new reference, up to the root.  A hash reference has a fixed size, so no ancestor's header
    changes.  (Nodes embedded in their parent are not chain nodes; `Gen.wrap` re-encodes a parent around one.)
    -> (new chain, new root)"""
    chain = list(chain)
    old, new = chain[j], new_node
    chain[j] = new
    for i in range(j - 1, -1, -1):
        parent = chain[i]
        href = hashref(keccak, old)
        assert parent.count(href) == 1, "node j is not referenced by its parent"
        chain[i] = parent.replace(href, hashref(keccak, new))
        old, new = parent, chain[i]
    return chain, keccak(chain[0])


class Gen:
    def __init__(self, keccak, seed=4242):
        self.k = keccak
        self.rng = np.random.default_rng(seed)
        self.cases = []
        self.off = 0  # bytes of node buffer emitted so far (for start residues)

    # -- small builders ------------------------------------------------------------------------------------------------
    def rand(self, n):
        return self.rng.integers(0, 256, n, dtype=np.uint8).tobytes()

    def nibs(self, n):
        return [int(x) for x in self.rng.integers(0, 16, n)]

    def href(self, node):
        return hashref(self.k, node)

    def branch(self, kids, value=b"\x80"):
        """17-item branch; kids: nibble -> encoded item; other slots random hash siblings or empty"""
        items = []
        for i in range(16):
            if i in kids:
                items.append(kids[i])
            elif self.rng.random() < 0.5:
                items.append(rlp_str(self.rand(32)))
            else:
                items.append(b"\x80")
        return rlp_list(items + [value])

    def full_branch(self, kids, value=b"\x80"):
        """all 16 slots hash references (532 bytes with an empty value)"""
        return rlp_list([kids.get(i, rlp_str(self.rand(32))) for i in range(16)] + [value])

    # -- placement -----------------------------------------------------------------------------------------------------
    @staticmethod
    def frames_for(depth, P):
        if depth == 0:
            return [] if P == 0 else None
        k = P - (depth - 1)
        if k < 1:
            return None
        return [("b",)] * (depth - 1) + [("b",) if k == 1 else ("e", k)]

    def wrap(self, frames, prefix, tail, embed):
        """ancestors over tail[0] along `frames`; -> (chain, root, chain index of the node under test or None)"""
        chain = list(tail)
        item = tail[0] if embed else self.href(tail[0])
        if embed:
            chain = chain[1:]
        pos = len(prefix)
        for f in reversed(frames):
            if f[0] == "b":
                pos -= 1
                node = self.branch({prefix[pos]: item})
            else:
                pos -= f[1]
                node = ext(prefix[pos:pos + f[1]], item)
            chain.insert(0, node)
            item = self.href(node)
        assert pos == 0
        return chain, self.k(chain[0]), (None if embed else len(frames))

    def emit(self, case, residue=None):
        if residue is not None and self.off % 16 != residue:  # a spacer proof (one junk node, REJECT by R1) in front
            s = (residue - self.off) % 16
            self.emit(Case("spacer", [self.rand(s)], bytes(32), self.k(b"spacer" + bytes([s])), REJECT, None, 0))
        self.check_linked(case)
        self.cases.append(case)
        self.off += sum(len(n) for n in case.nodes)

    def check_linked(self, c):
        """the walk really reaches the node under test: the root names node 0 and each node down to it names the next"""
        if c.name == "spacer" or not c.nodes:
            return
        assert self.k(c.nodes[0]) == c.root, c.name
        upto = c.target if c.target is not None else 0
        for i in range(1, upto + 1):
            assert self.href(c.nodes[i]) in c.nodes[i - 1], (c.name, i)

    def place(self, name, core, need_rest=None, depths=(0, 1, 5), embed=True, residue=None):
        """run `core(R, last)` -> (tail, status, value) or None at every placement and emit the cases"""
        for depth in depths:
            P = (64 - need_rest) if need_rest is not None else (depth if depth < 5 else 7)
            frames = self.frames_for(depth, P)
            if frames is None:
                continue
            for last in (True, False):
                prefix, R = self.nibs(P), self.nibs(64 - P)
                out = core(R, last)
                if out is None:
                    continue
                tail, st, val = out
                chain, root, t = self.wrap(frames, prefix, tail, False)
                self.emit(Case(f"{name}/d{depth}/{'last' if last else 'mid'}", chain, key_bytes(prefix + R), root, st, val, t),
                          residue if depth == 0 else None)
        if not embed:
            return
        P = (64 - need_rest) if need_rest is not None else 2
        frames = self.frames_for(2, P)
        if frames is None:
            return
        for last in (True, False):
            prefix, R = self.nibs(P), self.nibs(64 - P)
            out = core(R, last)
            if out is None:
                continue
            tail, st, val = out
            if len(tail[0]) >= 32 or tail[0][0] < 0xc0:
                continue
            chain, root, t = self.wrap(frames, prefix, tail, True)
            self.emit(Case(f"{name}/embedded/{'last' if last else 'mid'}", chain, key_bytes(prefix + R), root, st, val, t))

    # -- tails with the prescribed status --------------------------------------------------------------------------------
    def filler(self):
        return leaf(self.nibs(3), b"filler")

    def terminal(self, node, st, val, last):
        """a node the walk decides at: as the last node st, followed by anything REJECT (a terminal must be last)"""
        return ([node], st, val) if last else ([node, self.filler()], REJECT, None)

    def bad(self, node, follow, last):
        """a node R2-R4 reject; when not last it is followed by the node its reference would lead to, so that a walk which
        wrongly accepted it would go on to a verdict of its own"""
        return ([node], REJECT, None) if last else ([node] + follow[0], REJECT, None)

    def nxt(self, node, follow, last):
        """a node whose reference for the key leads on: last -> REJECT (a hash reference needs a node), else the follower's"""
        return ([node], REJECT, None) if last else ([node] + follow[0], follow[1], follow[2])

    def follow_leaf(self, R):
        v = self.rand(int(self.rng.choice([1, 7, 40])))
        return ([leaf(R, v)], PRESENT, v)


def build(keccak, seed=4242, damage_cases=1500):
    g = Gen(keccak, seed)
    named(g)
    random_damage(g, damage_cases)
    if g.off % 16:  # the corpus tiles without changing any node's start residue
        g.emit(Case("spacer", [g.rand(16 - g.off % 16)], bytes(32), keccak(b"spacer-end"), REJECT, None, 0))
    return g.cases


# ---------------------------------------------------------------------------------------------------------------------
def named(g):
    k = g.k

    def val(n):
        return g.rand(n) if n != 1 else bytes([0x80 | int(g.rng.integers(0, 128))])

    # ---- RLP framing -----------------------------------------------------------------------------------------------
    def leaf_long_hdr(pay_target):
        def core(R, last):
            hp = rlp_str(_hp(R, True))
            vl = pay_target - len(hp) - 1
            if vl < 2 or vl > 55:
                return None
            v = val(vl)
            pay = hp + rlp_str(v)
            if len(pay) != pay_target:
                return None
            node = long_list(pay)
            st = PRESENT if pay_target > 55 else REJECT
            return g.terminal(node, st, v, last) if st == PRESENT else g.bad(node, ([], 0, None), last)
        return core
    for t in (40, 55, 56, 57):
        g.place(f"framing/leaf_long_header_pay{t}", leaf_long_hdr(t))

    def branch_variant(encode_mut, kids_n=1, status_ok=False):
        """a simple branch (kids_n hash children, one at the key's nibble) re-encoded by encode_mut; the follower is a leaf"""
        def core(R, last):
            fol = g.follow_leaf(R[1:])
            kids = {R[0]: g.href(fol[0][0])}
            others = [i for i in range(16) if i != R[0]]
            for i in g.rng.choice(others, kids_n - 1, replace=False):
                kids[int(i)] = rlp_str(g.rand(32))
            items = [kids.get(i, b"\x80") for i in range(16)] + [b"\x80"]
            node = encode_mut(items)
            if node is None:
                return None
            return g.nxt(node, fol, last) if status_ok else g.bad(node, fol, last)
        return core

    # a simple branch under a long header with payload <= 55 (1 hash child: payload 49)
    g.place("framing/branch_long_header_pay49", branch_variant(lambda it: long_list(b"".join(it)), 1), embed=False)
    g.place("framing/branch_long_header_pay81_ok", branch_variant(lambda it: long_list(b"".join(it)), 2, True), embed=False)
    # a zero first length byte: 0xf9 00 LL (payload < 256) and 0xf8 00 (never canonical)
    g.place("framing/branch_zero_len_byte_f9", branch_variant(lambda it: long_list(b"".join(it), n_len=2), 3), embed=False)
    g.place("summary/f9_header_pay_lt256", branch_variant(lambda it: long_list(b"".join(it), n_len=2), 5), embed=False)
    g.place("framing/leaf_zero_len_byte_f9",
            lambda R, last: g.bad(long_list(rlp_str(_hp(R, True)) + rlp_str(val(70)), n_len=2), ([], 0, None), last))
    g.place("framing/value_zero_len_byte_b9",
            lambda R, last: g.bad(rlp_list([rlp_str(_hp(R, True)), b"\xb9\x00\x40" + g.rand(64)]), ([], 0, None), last))
    g.place("framing/value_long_header_le55",
            lambda R, last: g.bad(rlp_list([rlp_str(_hp(R, True)), b"\xb8\x37" + g.rand(55)]), ([], 0, None), last))

    def value_long_header_56(R, last):  # the shortest string the long form is right for
        v = g.rand(56)
        return g.terminal(rlp_list([rlp_str(_hp(R, True)), b"\xb8\x38" + v]), PRESENT, v, last)
    g.place("framing/value_long_header_56_ok", value_long_header_56)
    # length-of-length 5 (list and string)
    g.place("framing/list_len_of_len5",
            lambda R, last: g.bad(long_list(rlp_str(_hp(R, True)) + rlp_str(val(60)), n_len=5), ([], 0, None), last), embed=False)
    g.place("framing/branch_len_of_len5", branch_variant(lambda it: long_list(b"".join(it), n_len=5), 3), embed=False)
    g.place("framing/string_len_of_len5",
            lambda R, last: g.bad(rlp_list([rlp_str(_hp(R, True)), b"\xbc\x00\x00\x00\x00\x40" + g.rand(64)]), ([], 0, None), last))

    # the declared length one more / one less than the node; a trailing byte after the list
    def relen(node, d):
        b = node[0]
        if b <= 0xf7:
            return bytes([b + d]) + node[1:]
        n = b - 0xf7
        L = int.from_bytes(node[1:1 + n], "big") + d
        return node[:1] + L.to_bytes(n, "big") + node[1 + n:]

    for vl, tag in ((5, "short"), (80, "long")):
        for d in (1, -1):
            g.place(f"framing/leaf_{tag}_declared{d:+d}",
                    lambda R, last, vl=vl, d=d: g.bad(relen(leaf(R, val(vl)), d), ([], 0, None), last))
        g.place(f"framing/leaf_{tag}_trailing_byte",
                lambda R, last, vl=vl: g.bad(leaf(R, val(vl)) + b"\x00", ([], 0, None), last))
    for d in (1, -1):
        g.place(f"framing/branch_declared{d:+d}", branch_variant(lambda it, d=d: relen(rlp_list(it), d), 4), embed=False)
    g.place("framing/branch_trailing_byte", branch_variant(lambda it: rlp_list(it) + b"\x80", 4), embed=False)
    # 0x81 xx with xx < 0x80 (a single byte that must encode as itself), and the canonical 0x81 xx >= 0x80
    for x in (0x00, 0x7f):
        g.place(f"framing/value_81_{x:02x}", lambda R, last, x=x: g.bad(rlp_list([rlp_str(_hp(R, True)), bytes([0x81, x])]), ([], 0, None), last))
    g.place("framing/value_81_80_ok", lambda R, last: g.terminal(rlp_list([rlp_str(_hp(R, True)), b"\x81\x80"]), PRESENT, b"\x80", last))
    g.place("framing/hp_81_single_nibble", lambda R, last: g.bad(rlp_list([b"\x81" + _hp(R, True), rlp_str(b"v")]), ([], 0, None), last),
            need_rest=1, depths=(1, 5))
    g.place("framing/value_81_in_branch_item",
            branch_variant(lambda it: rlp_list(it[:-1] + [b"\x81\x05"]), 2))
    # a string that should be a list, a list that should be a string
    g.place("framing/node_is_string", lambda R, last: g.bad(rlp_str(payload_of(leaf(R, val(9)))), ([], 0, None), last))
    g.place("framing/hp_is_list", lambda R, last: g.bad(rlp_list([rlp_list([rlp_str(_hp(R, True))]), rlp_str(b"v")]), ([], 0, None), last))
    g.place("leaf/value_is_list", lambda R, last: g.bad(rlp_list([rlp_str(_hp(R, True)), rlp_list([rlp_str(b"v")])]), ([], 0, None), last))
    g.place("leaf/value_empty", lambda R, last: g.terminal(leaf(R, b""), PRESENT, b"", last))
    g.place("framing/empty_list", lambda R, last: g.bad(b"\xc0", ([], 0, None), last))
    g.place("framing/empty_node", lambda R, last: g.bad(b"", ([], 0, None), last), embed=False)

    # ---- branch ------------------------------------------------------------------------------------------------------
    g.place("branch/16_items", branch_variant(lambda it: rlp_list(it[:16]), 3))
    g.place("branch/18_items", branch_variant(lambda it: rlp_list(it + [b"\x80"]), 3))
    g.place("branch/2_items_not_leaf", branch_variant(lambda it: rlp_list(it[:2]) if it[0] == b"\x80" else None, 1))
    for n in (31, 33, 1, 20):
        def child_len(R, last, n=n):  # the key's child is a string of n bytes: only 0 or 32 are references
            node = g.branch({R[0]: rlp_str(g.rand(n))})
            return g.bad(node, g.follow_leaf(R[1:]), last)
        g.place(f"branch/child_string_{n}", child_len)

        def other_len(R, last, n=n):  # another slot holds it: the walk reads only the key's child
            fol = g.follow_leaf(R[1:])
            other = (R[0] + 1 + int(g.rng.integers(0, 15))) % 16
            return g.nxt(g.branch({R[0]: g.href(fol[0][0]), other: rlp_str(g.rand(n))}), fol, last)
        g.place(f"branch/other_child_string_{n}", other_len, embed=False)

    # embedded children of exactly 31 and 32 bytes (a leaf walked in place; 32 bytes must have been a hash reference)
    def embedded_leaf(total, present):
        def core(R, last):
            path = R[1:] if present else R[1:][:len(R) - 2]
            for vl in range(0, 40):
                c = leaf(path, g.rand(vl))
                if len(c) == total:
                    break
            else:
                return None
            node = g.branch({R[0]: c})
            if total >= 32:
                return g.bad(node, ([g.filler()], 0, None), last)
            if present:
                v = c[len(c) - vl:] if vl else b""
                return g.terminal(node, PRESENT, v, last)
            return g.terminal(node, ABSENT, None, last)
        return core
    for total in (31, 32):
        g.place(f"branch/embedded_leaf_{total}_present_path", embedded_leaf(total, True), need_rest=12)
        g.place(f"branch/embedded_leaf_{total}_short_path", embedded_leaf(total, False), need_rest=12)
        g.place(f"branch/embedded_leaf_{total}_low", embedded_leaf(total, False))

    # an embedded child that is itself malformed (walked in place by the same rules)
    def embedded_bad(mut):
        def core(R, last):
            c = mut(leaf(R[1:], b"ab"))
            return g.bad(g.branch({R[0]: c}), ([g.filler()], 0, None), last)
        return core
    g.place("branch/embedded_child_16_items", embedded_bad(lambda c: rlp_list([b"\x80"] * 16)), need_rest=8)
    g.place("branch/embedded_child_string_hp", embedded_bad(lambda c: rlp_list([rlp_list([b"\x20"]), b"\x01"])), need_rest=8)
    g.place("branch/embedded_child_flag4", embedded_bad(lambda c: c[:2] + bytes([0x40 | (c[2] & 15)]) + c[3:] if c[1] >= 0x80 else None), need_rest=8)
    g.place("branch/embedded_child_value_list", embedded_bad(lambda c: rlp_list([rlp_str(b"\x20"), rlp_list([])])), need_rest=1)
    # an embedded extension (short path, embedded leaf under it), and an empty branch slot
    def embedded_ext(R, last):
        v = g.rand(3)
        inner = leaf(R[3:], v)
        e = ext(R[1:3], inner)
        if len(e) >= 32:
            return None
        return g.terminal(g.branch({R[0]: e}), PRESENT, v, last)
    g.place("branch/embedded_ext_embedded_leaf", embedded_ext, need_rest=8)

    def empty_slot(R, last):
        node = g.branch({R[0]: b"\x80", (R[0] + 1) % 16: rlp_str(g.rand(32))})
        return g.terminal(node, ABSENT, None, last)
    g.place("branch/empty_slot", empty_slot)
    # a hash child when the chain ends there (last) / followed (mid)
    g.place("branch/hash_child", branch_variant(lambda it: rlp_list(it), 6, True))
    # a non-empty value with the key not exhausted: the walk goes on to the child
    for vv in (b"\x00", b"\x81\x80", rlp_str(b"value"), rlp_str(bytes(60))):
        g.place(f"branch/value_{vv[:2].hex()}_key_not_exhausted", branch_variant(lambda it, vv=vv: rlp_list(it[:-1] + [vv]), 4, True))
    g.place("branch/value_list_key_not_exhausted", branch_variant(lambda it: rlp_list(it[:-1] + [b"\xc0"]), 4, True))

    # the key exhausted at a branch, through an extension over the rest of the key (64 nibbles at depth 0)
    def exhausted(value_item, st, v, hashed_kids):
        def core(R, last):
            kids = {i: rlp_str(g.rand(32)) for i in range(16) if hashed_kids and g.rng.random() < 0.6}
            b = rlp_list([kids.get(i, b"\x80") for i in range(16)] + [value_item])
            e = ext(R, g.href(b))
            if not last:  # the branch is the last node here; "mid" puts one more node behind it
                return ([e, b, g.filler()], REJECT, None)
            return ([e, b], st, v)
        return core
    for hk in (False, True):
        g.place(f"branch/key_exhausted_value_empty_hk{int(hk)}", exhausted(b"\x80", ABSENT, None, hk))
        g.place(f"branch/key_exhausted_value_present_hk{int(hk)}", exhausted(rlp_str(b"xyz"), PRESENT, b"xyz", hk))
        g.place(f"branch/key_exhausted_value_list_hk{int(hk)}", exhausted(rlp_list([b"\x01"]), REJECT, None, hk))

    # ---- summary near-misses ---------------------------------------------------------------------------------------
    # a 532-byte node with one 0xa0 child replaced by a 33-byte list (0xe0 + 32 bytes): the list's bytes are the follower's
    # hash, so a walk that took the node for a simple branch would go on to a verdict
    for c in (0, 7, 15):
        def near532(R, last, c=c):
            fol = g.follow_leaf(R[1:])
            if R[0] == c:
                node = g.full_branch({c: b"\xe0" + k(fol[0][0])})
                assert len(node) == 532
                return g.bad(node, fol, last)
            node = g.full_branch({c: b"\xe0" + g.rand(32), R[0]: g.href(fol[0][0])})
            return g.nxt(node, fol, last)
        g.place(f"summary/532_child{c}_list_e0", near532, embed=False)

        def near532_at(R, last, c=c):  # the same with the key's nibble forced onto the list
            R = [c] + R[1:]
            fol = g.follow_leaf(R[1:])
            return g.bad(g.full_branch({c: b"\xe0" + k(fol[0][0])}), fol, last)
        g.place(f"summary/532_child{c}_list_e0_on_key", near532_at, embed=False)

    def full_branch_on(value):
        """a branch with 16 hash children and `value`; the key's child leads to a leaf (532 bytes with an empty value)"""
        def core(R, last):
            fol = g.follow_leaf(R[1:])
            return g.nxt(g.full_branch({R[0]: g.href(fol[0][0])}, value), fol, last)
        return core
    for vv in (b"\x00", b"\x81\x80"):
        g.place(f"summary/full_branch_value_{vv.hex()}", full_branch_on(vv), embed=False)
        g.place(f"summary/branch_value_{vv.hex()}", branch_variant(lambda it, vv=vv: rlp_list(it[:-1] + [vv]), 3, True), embed=False)
    g.place("summary/full_branch_532", full_branch_on(b"\x80"), embed=False)
    # the key exhausted at a simple branch: the summary's fast path must not run (there is no next nibble)
    g.place("summary/simple_branch_at_key_end", exhausted(b"\x80", ABSENT, None, True), need_rest=5, depths=(1, 5))
    # a simple branch with every number of hash children (the summary's scan), key on a hash child and on an empty slot
    for kn in range(0, 17):
        def simple(R, last, kn=kn):
            if kn == 0:
                return g.terminal(rlp_list([b"\x80"] * 17), ABSENT, None, last)
            fol = g.follow_leaf(R[1:])
            kids = {R[0]: g.href(fol[0][0])}
            for i in g.rng.permutation([i for i in range(16) if i != R[0]])[:kn - 1]:
                kids[int(i)] = rlp_str(g.rand(32))
            return g.nxt(rlp_list([kids.get(i, b"\x80") for i in range(16)] + [b"\x80"]), fol, last)
        g.place(f"summary/simple_branch_{kn}_hash_children", simple, embed=False)

    # ---- leaf and extension -----------------------------------------------------------------------------------------
    # hex-prefix flags 0-15 over a leaf's hex-prefix bytes, even and odd path
    for parity in (0, 1):
        for f in range(16):
            def flagged(R, last, f=f):
                v = g.rand(5)
                hp = bytearray(_hp(R, True))
                hp[0] = (f << 4) | (hp[0] & 15)
                node = rlp_list([rlp_str(bytes(hp)), rlp_str(v)])
                r = len(R)
                if f > 3:
                    return g.bad(node, ([], 0, None), last)
                odd = f & 1
                if not odd and (hp[0] & 15):
                    return g.bad(node, ([], 0, None), last)
                plen = 2 * (len(hp) - 1) + odd
                path = ([hp[0] & 15] if odd else []) + [n for b in hp[1:] for n in (b >> 4, b & 15)]
                if plen > 64:
                    return g.bad(node, ([], 0, None), last)
                match = path == R[:plen]
                if f & 2:
                    st = PRESENT if (match and plen == r) else ABSENT
                    return g.terminal(node, st, v if st == PRESENT else None, last)
                # extension: its child is the 5-byte value string (not a reference)
                if plen == 0 or (match and plen <= r):
                    return g.bad(node, ([], 0, None), last)
                return g.terminal(node, ABSENT, None, last)
            g.place(f"leaf/hp_flag_{f}_{'odd' if parity else 'even'}", flagged, need_rest=10 + parity, depths=(1, 5))
            if parity == 0:
                g.place(f"leaf/hp_flag_{f}_d0", flagged, embed=False, depths=(0,))
    # an even path with a non-zero pad; an empty hex-prefix string
    for fl in (0x20, 0x00):
        for pad in (1, 8, 15):
            def padded(R, last, fl=fl, pad=pad):
                hp = bytearray(_hp(R, fl == 0x20))
                hp[0] = fl | pad
                fol = g.follow_leaf([])
                node = rlp_list([rlp_str(bytes(hp)), rlp_str(g.rand(4)) if fl else g.href(fol[0][0])])
                return g.bad(node, fol, last)
            g.place(f"leaf/even_path_pad_{fl >> 4}_{pad}", padded, need_rest=6)
    g.place("leaf/empty_hp", lambda R, last: g.bad(rlp_list([b"\x80", rlp_str(b"vv")]), ([], 0, None), last))

    def ext_empty_hp(R, last):
        fol = g.follow_leaf(R)
        return g.bad(rlp_list([b"\x80", g.href(fol[0][0])]), fol, last)
    g.place("ext/empty_hp", ext_empty_hp)

    # leaf path lengths 0-64 (ending the key, and one short / one long of it), 65 and 66
    for L in range(0, 67):
        def sweep(R, last, L=L):
            v = g.rand(int(g.rng.choice([1, 3, 33])))
            if L > 64:
                hp = bytes([0x30 | g.nibs(1)[0]]) + g.rand(32) if L == 65 else b"\x20" + g.rand(33)
                return g.bad(rlp_list([rlp_str(hp), rlp_str(v)]), ([], 0, None), last)
            return g.terminal(leaf(R, v), PRESENT, v, last)
        g.place(f"leaf/path_len_{L}", sweep, need_rest=min(L, 64), depths=(0, 1, 5), embed=L <= 20)

        def off_by(R, last, L=L):  # a leaf of L nibbles where the key has L +- 1 left
            if L == 0 or L > 64:
                return None
            path = R[:-1] if len(R) > L else R + [g.nibs(1)[0]]
            return g.terminal(leaf(path, b"v"), ABSENT, None, last)
        if 0 < L <= 64:
            g.place(f"leaf/path_len_{L}_short", off_by, need_rest=L + 1 if L < 64 else None, depths=(0, 1, 5) if L < 64 else (), embed=False)
        if 1 < L <= 64:
            g.place(f"leaf/path_len_{L}_long", off_by, need_rest=L - 1, depths=(1, 5), embed=False)

    # a mismatch at every nibble of the path, both parities (a leaf that does end the key, one nibble wrong)
    for r in (63, 64, 33, 32, 5, 4, 2, 1):
        for j in range(r):
            def miss(R, last, j=j):
                path = list(R)
                path[j] ^= 1 + int(g.rng.integers(0, 15))
                return g.terminal(leaf(path, g.rand(3)), ABSENT, None, last)
            g.place(f"leaf/mismatch_r{r}_at_{j}", miss, need_rest=r, depths=(0,) if r == 64 else (5,), embed=False)

    # extensions: empty path, empty child, path longer than the rest of the key, under an extension, every length

    def ext_empty_path(R, last):
        fol = g.follow_leaf(R)
        return g.bad(ext([], g.href(fol[0][0])), fol, last)
    g.place("ext/empty_path", ext_empty_path)
    g.place("ext/empty_child", lambda R, last: g.bad(ext(R[:2], b"\x80"), ([g.filler()], 0, None), last))
    g.place("ext/child_string_31", lambda R, last: g.bad(ext(R[:2], rlp_str(g.rand(31))), ([g.filler()], 0, None), last))
    g.place("ext/path_longer_than_key", lambda R, last: g.terminal(ext(R + g.nibs(1), rlp_str(g.rand(32))), ABSENT, None, last),
            need_rest=9)
    g.place("ext/path_diverges", lambda R, last: g.terminal(ext([R[0] ^ 1] + R[1:3], rlp_str(g.rand(32))), ABSENT, None, last))
    g.place("ext/path_65", lambda R, last: g.bad(rlp_list([rlp_str(bytes([0x10]) + g.rand(32)), rlp_str(g.rand(32))]), ([], 0, None), last))

    def ext_ext(R, last):
        fol = g.follow_leaf(R[4:])
        inner = ext(R[2:4], g.href(fol[0][0]))
        outer = ext(R[:2], g.href(inner))
        return g.nxt(outer, ([inner] + fol[0], fol[1], fol[2]), last)
    g.place("ext/under_ext", ext_ext)

    def ext_ext_embedded(R, last):
        v = g.rand(2)
        inner = ext(R[2:3], leaf(R[3:], v))
        if len(inner) >= 32:
            return None
        return g.terminal(ext(R[:2], inner), PRESENT, v, last)
    g.place("ext/under_ext_embedded", ext_ext_embedded, need_rest=12)
    for L in (1, 2, 3, 31, 32, 33, 62, 63):
        def ext_len(R, last, L=L):
            fol = g.follow_leaf(R[L:])
            return g.nxt(ext(R[:L], g.href(fol[0][0])), fol, last)
        g.place(f"ext/path_len_{L}", ext_len, need_rest=64 if L > 60 else None, depths=(0,) if L > 60 else (0, 1, 5), embed=False)

    # ---- R4: the empty chain ----------------------------------------------------------------------------------------
    for root, st in ((EMPTY_ROOT, ABSENT), (g.rand(32), REJECT)):
        g.emit(Case(f"r4/empty_chain_{'empty_root' if st == ABSENT else 'other_root'}", [], key_bytes(g.nibs(64)), root, st, None, None))

    # ---- sizes and placement ----------------------------------------------------------------------------------------
    def sized_leaf(N):
        def core(R, last):
            hp = rlp_str(_hp(R, True))
            for vl in range(max(0, N - len(hp) - 10), N):
                v = g.rand(vl)
                node = rlp_list([hp, rlp_str(v)])
                if len(node) == N:
                    return g.terminal(node, PRESENT, v, last)
                if len(node) > N:
                    return None
            return None
        return core

    def sized_branch(N):
        """a branch of N bytes: hash children plus a value that fills it; the key's child leads to a leaf"""
        def core(R, last):
            fol = g.follow_leaf(R[1:])
            kids = {R[0]: g.href(fol[0][0])}
            for i in range(16):
                if i != R[0] and g.rng.random() < 0.5:
                    kids[i] = rlp_str(g.rand(32))
            body = b"".join(kids.get(i, b"\x80") for i in range(16))
            for vl in range(max(0, N - len(body) - 10), N):
                node = rlp_list([kids.get(i, b"\x80") for i in range(16)] + [rlp_str(g.rand(vl))])
                if len(node) == N:
                    return g.nxt(node, fol, last)
                if len(node) > N:
                    return None
            return None
        return core
    sizes = [20, 31, 32, 40, 55, 56, 57, 100, 135, 136, 137, 271, 272, 273, 408, 532] + list(range(544, 562)) + [600, 4095, 4096, 4097, 70000]
    for N in sizes:
        g.place(f"size/leaf_{N}", sized_leaf(N), need_rest=8 if N < 45 else None, embed=N < 32)
        if N >= 140:
            g.place(f"size/branch_{N}", sized_branch(N), embed=False)
    # every start residue mod 16, for nodes around the rate block and the staging window
    for N in (136, 137, 272, 532, 545, 548, 552, 556, 560, 561, 4096):
        for res in range(16):
            g.place(f"residue/leaf_{N}_at_{res}", sized_leaf(N), depths=(0,), embed=False, residue=res)
            if N in (532, 545, 560):
                g.place(f"residue/branch_{N}_at_{res}", sized_branch(N) if N != 532 else full_branch_on(b"\x80"),
                        depths=(0,), embed=False, residue=res)


def random_damage(g, n):
    """test_fuzz_walk.damage applied to one node of a genuine proof, then resealed: byte-level damage that reaches R2-R4"""
    from test_fuzz_walk import damage
    from oracle_lib import get
    o = get()
    rng = np.random.default_rng(g.rng.integers(1 << 30))
    proofs = []
    for vmax in (1, 33, 140, 600, 1200):
        keys = sorted(rng.integers(0, 256, 32, dtype=np.uint8).tobytes() for _ in range(48))
        kv = [(kk, rng.integers(0, 256, int(rng.integers(1, vmax + 1)), dtype=np.uint8).tobytes()) for kk in keys]
        t = o.trie(kv)
        proofs += [(t.prove(kk), kk, t.root()) for kk in keys[:32]]
        proofs += [(t.prove(kk), kk, t.root()) for kk in (rng.integers(0, 256, 32, dtype=np.uint8).tobytes() for _ in range(8))]
    made = 0
    while made < n:
        nl, key, root = proofs[int(rng.integers(0, len(proofs)))]
        if not nl:
            continue
        j = int(rng.integers(0, len(nl)))
        d = damage(([nl[j]], key, root), rng)
        if len(d[0]) != 1 or d[1] != key or d[2] != root or d[0][0] == nl[j]:
            continue
        chain, new_root = reseal(g.k, nl, j, d[0][0])
        g.emit(Case("damage", chain, key, new_root, None, None, j))
        made += 1
