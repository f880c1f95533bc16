"""The rules of entry point T (state transition roots, DESIGN.md "T: state transition roots") stated on the CPU for the tests,
written from the header's statement, not from the device code: expand the witness along the listed keys, apply the diff, and
rebuild each trie with the off-path children the witness only references (stubs) kept as they are or moved up.  Also builds
the witnesses the CPU and GPU tests share.  TEST INFRASTRUCTURE: the product never imports this."""
import numpy as np

import oracle_lib
from helpers import _hp, rlp_int_be, rlp_list, rlp_str
from resident_state_model import CLEAR, DELETE, ZERO32
from state_read_oracle import _item, decode_account

EMPTY_ROOT = bytes.fromhex("56e81f171bcc55a6ff8345e692c0f86e5b48e01b996cadc001622fb5e363b421")
BAD, MISSING = 1, 2


def nibbles(key):
    return tuple(n for b in key for n in (b >> 4, b & 15))


def decode(node):
    """-> ("leaf", path, value) / ("ext", path, child) / ("branch", [16 children]) or None when the node breaks R2-R4;
    a child is None (empty), ("hash", 32 bytes) or ("embed", node bytes)"""
    top = _item(node, 0, len(node))
    if top is None or not top[0] or top[2] != len(node):
        return None
    items, pos = [], top[1]
    while pos < top[2]:
        it = _item(node, pos, top[2])
        if it is None or len(items) == 17:
            return None
        items.append((it, pos))
        pos = it[2]

    def child(it, pos):
        is_list, a, b = it
        if is_list:
            return ("embed", node[pos:b]) if b - pos < 32 else False
        if b == a:
            return None
        return ("hash", node[a:b]) if b - a == 32 else False

    if len(items) == 17:
        kids = [child(*items[v]) for v in range(16)]
        (is_list, a, b), _ = items[16]
        if False in kids or is_list or b != a:
            return None
        return ("branch", kids)
    if len(items) != 2:
        return None
    (is_list, a, b), _ = items[0]
    if is_list or b == a:
        return None
    hp = node[a:b]
    flag = hp[0] >> 4
    if flag > 3 or (not flag & 1 and hp[0] & 15):
        return None
    path = ((hp[0] & 15,) if flag & 1 else ()) + nibbles(hp[1:])
    if len(path) > 64:
        return None
    if flag & 2:
        (is_list, a, b), _ = items[1]
        return None if is_list else ("leaf", path, node[a:b])
    c = child(*items[1])
    if not path or not c:
        return None
    return ("ext", path, c)


class Run:
    """one block: the node table, the digests looked up, and the status flags"""

    def __init__(self, keccak, table):
        self.keccak, self.table, self.reads, self.flags = keccak, table, set(), 0
        self.collapses = []  # per moved stub: "branch" (known below an extension, or looked up), "leaf" or "ext"

    def lookup(self, h):
        self.reads.add(h)
        n = self.table.get(h)
        if n is None:
            self.flags |= MISSING
        return n

    def expand(self, root, keys):
        """the witness along the sorted 64-nibble `keys` under `root` -> (leaves {key: value}, stubs [(prefix, ref, below_ext)])"""
        leaves, stubs = {}, []

        def visit(ref, node, prefix, ks, below_ext):
            if node is None:
                if not ks:
                    stubs.append((prefix, ref, below_ext))
                    return
                node = self.lookup(ref)
                if node is None:
                    return
            t = decode(node)
            if t is None:
                self.flags |= BAD
                return
            d = len(prefix)
            if t[0] == "leaf":
                if d + len(t[1]) != 64:
                    self.flags |= BAD
                else:
                    leaves[prefix + t[1]] = t[2]
                return
            if t[0] == "ext":
                if d + len(t[1]) >= 64:
                    self.flags |= BAD
                    return
                p = prefix + t[1]
                kids = [(p, t[2], [k for k in ks if k[:len(p)] == p], True)]
            else:
                if d >= 64:
                    self.flags |= BAD
                    return
                kids = [(prefix + (v,), c, [k for k in ks if k[d] == v], False) for v, c in enumerate(t[1]) if c is not None]
            for p, c, sub, bx in kids:
                visit(c[1] if c[0] == "hash" else None, c[1] if c[0] == "embed" else None, p, sub, bx)

        if root != EMPTY_ROOT:
            visit(root, None, (), keys, False)
        return leaves, stubs

    def moved(self, prefix, ref, below_ext, pl):
        """the node a stub at depth len(prefix) becomes at depth pl < len(prefix)"""
        head = prefix[pl:]
        if below_ext:
            self.collapses.append("branch")
        else:
            node = self.lookup(ref)
            if node is None:
                return None
            t = decode(node)
            if t is None:
                self.flags |= BAD
                return None
            self.collapses.append(t[0])
            if t[0] == "leaf":
                if len(prefix) + len(t[1]) != 64:
                    self.flags |= BAD
                    return None
                return rlp_list([rlp_str(_hp(head + t[1], True)), rlp_str(t[2])])
            if t[0] == "ext":
                if len(prefix) + len(t[1]) >= 64:
                    self.flags |= BAD
                    return None
                c = t[2]
                return rlp_list([rlp_str(_hp(head + t[1], False)), rlp_str(c[1]) if c[0] == "hash" else c[1]])
        return rlp_list([rlp_str(_hp(head, False)), rlp_str(ref)])

    def rebuild(self, leaves, stubs):
        """-> the root of the trie holding `leaves` and the stubs (hashed references), or None when a rule fails"""
        items = [(k, ("leaf", v)) for k, v in leaves.items()]
        items += [(p + (0,) * (64 - len(p)), ("stub", p, r, bx)) for p, r, bx in stubs]
        items.sort(key=lambda x: x[0])
        fixed = {}
        for i, (k, it) in enumerate(items):
            if it[0] != "stub":
                continue
            pl = 0
            for j in (i - 1, i + 1):
                if 0 <= j < len(items):
                    o = items[j][0]
                    c = 0
                    while c < 64 and o[c] == k[c]:
                        c += 1
                    pl = max(pl, c + 1)
            _, p, r, bx = it
            assert pl <= len(p)
            if pl == len(p):
                fixed[i] = b"\xa0" + r
                continue
            enc = self.moved(p, r, bx, pl)
            if enc is None:
                continue
            if len(enc) < 32:
                self.flags |= BAD
                continue
            fixed[i] = b"\xa0" + self.keccak(enc)
        if self.flags:
            return None
        kc = self.keccak

        def ref(node):
            return node if len(node) < 32 else rlp_str(kc(node))

        def build(lo, hi, level):
            """-> ("ref", reference) for a stub that hangs here, else ("node", RLP)"""
            if hi - lo == 1:
                k, it = items[lo]
                if it[0] == "stub":
                    return ("ref", fixed[lo])
                return ("node", rlp_list([rlp_str(_hp(k[level:], True)), rlp_str(it[1])]))
            a, b = items[lo][0], items[hi - 1][0]
            c = level
            while a[c] == b[c]:
                c += 1
            br = build_branch(lo, hi, c)
            if c > level:
                return ("node", rlp_list([rlp_str(_hp(a[level:c], False)), ref(br)]))
            return ("node", br)

        def build_branch(lo, hi, c):
            slots = []
            i = lo
            for v in range(16):
                j = i
                while j < hi and items[j][0][c] == v:
                    j += 1
                if j == i:
                    slots.append(rlp_str(b""))
                else:
                    kind, x = build(i, j, c + 1)
                    slots.append(x if kind == "ref" else ref(x))
                i = j
            return rlp_list(slots + [rlp_str(b"")])

        if not items:
            return EMPTY_ROOT
        kind, x = build(0, len(items), 0)
        return x[1:] if kind == "ref" else kc(x)


def account_leaf(nonce, balance, sroot, code_hash):
    return rlp_list([rlp_int_be(int(nonce).to_bytes(8, "big")), rlp_int_be(balance), rlp_str(sroot), rlp_str(code_hash)])


def transition(oracle, node_list, pre_root, diff, collapses=None):
    """one block: diff (resident_state_model.Diff) applied to the witness `node_list` under `pre_root` ->
    (status, root or None, [storage root per listed account], reads: the digests the computation looked up); `collapses`
    (a list, optional) receives the kind of node each moved stub turned out to be"""
    kc = oracle.keccak256
    run = Run(kc, {kc(n): n for n in node_list})
    if collapses is not None:
        run.collapses = collapses
    accs = diff.accounts
    # stage 1: P's account walk from the block's root
    acc_state = []
    if accs:
        data, off = oracle_lib.csr(list(node_list), np.uint64)
        keys = np.frombuffer(b"".join(a[0] for a in accs), np.uint8).copy()
        roots = np.frombuffer(pre_root * len(accs), np.uint8).copy()
        st, vo, vl = oracle.verify_bag(np.concatenate([data, np.zeros(64, np.uint8)]), off, keys, roots)
        for i in range(len(accs)):
            s, sroot = int(st[i]), EMPTY_ROOT
            if s == 1:
                body = decode_account(data[int(vo[i]):int(vo[i]) + int(vl[i])].tobytes())
                s, sroot = (0, EMPTY_ROOT) if body is None else (1, body[2])
            run.flags |= BAD if s == 0 else MISSING if s == 3 else 0
            acc_state.append((s, sroot))
    if run.flags:
        return status_of(run.flags), None, [ZERO32] * len(accs), run.reads
    # stage 2: expand every segment along its listed keys
    segs = []
    for i, (key, flags, nonce, bal, ch) in enumerate(accs):
        if flags & DELETE:
            continue
        s, sroot = acc_state[i]
        root = EMPTY_ROOT if (flags & CLEAR or s != 1) else sroot
        writes = {sk: v for ai, sk, v in diff.slots if ai == i}
        segs.append((i, root, writes))
    expanded = []
    for i, root, writes in segs:
        expanded.append(run.expand(root, sorted(nibbles(k) for k in writes)))
    acc_exp = run.expand(pre_root, sorted(nibbles(a[0]) for a in accs))
    if run.flags:
        return status_of(run.flags), None, [ZERO32] * len(accs), run.reads
    # stage 3: apply, place the stubs, rebuild
    sroots = [ZERO32] * len(accs)
    for (i, _, writes), (leaves, stubs) in zip(segs, expanded):
        for sk, v in writes.items():
            if v == ZERO32:
                leaves.pop(nibbles(sk), None)
            else:
                leaves[nibbles(sk)] = rlp_str(v.lstrip(b"\x00"))
        sroots[i] = run.rebuild(leaves, stubs)
    leaves, stubs = acc_exp
    for i, (key, flags, nonce, bal, ch) in enumerate(accs):
        if flags & DELETE:
            leaves.pop(nibbles(key), None)
        else:
            leaves[nibbles(key)] = account_leaf(nonce, bal, sroots[i] or ZERO32, ch)
    root = run.rebuild(leaves, stubs)
    if run.flags:
        return status_of(run.flags), None, [ZERO32] * len(accs), run.reads
    return 1, root, sroots, run.reads


def status_of(flags):
    return 0 if flags & BAD else 3 if flags & MISSING else 1


# ---- witnesses: what a geth-style witness of a block holds -------------------------------------------------------------------
def witness(oracle, model, diff, account_trie=None):
    """the pre-state proofs of every key the diff lists (accounts, and slots of accounts present, not deleted and not cleared),
    plus the proofs of the nearest surviving neighbours of each key the diff deletes -- the nodes of `model` (a StateModel).
    account_trie: the model's account trie when the caller already built it (many blocks over one large state)"""
    nodes = {}
    acc_keys = sorted(model.acc)
    if not acc_keys:
        return []
    trie = account_trie or oracle.trie([(k, model.leaf(k)) for k in acc_keys])

    def prove(t, keys, k):
        for nd in t.prove(k):
            nodes[nd] = 1

    def neighbours(t, keys, gone, k):
        import bisect
        i = bisect.bisect_left(keys, k)
        for j, step in ((i - 1, -1), (i + (1 if i < len(keys) and keys[i] == k else 0), 1)):
            while 0 <= j < len(keys) and keys[j] in gone:
                j += step
            if 0 <= j < len(keys):
                prove(t, keys, keys[j])

    gone = {a[0] for a in diff.accounts if a[1] & DELETE}
    for a in diff.accounts:
        prove(trie, acc_keys, a[0])
        if a[1] & DELETE:
            neighbours(trie, acc_keys, gone, a[0])
    for ai, (key, flags, *_rest) in enumerate(diff.accounts):
        acc = model.acc.get(key)
        if acc is None or flags & (DELETE | CLEAR) or not acc.storage:
            continue
        ks = sorted(acc.storage)
        st = oracle.trie([(k, rlp_str(acc.storage[k].lstrip(b"\x00"))) for k in ks])
        writes = [(sk, v) for i, sk, v in diff.slots if i == ai]
        sgone = {sk for sk, v in writes if v == ZERO32}
        for sk, v in writes:
            prove(st, ks, sk)
            if v == ZERO32:
                neighbours(st, ks, sgone, sk)
    return list(nodes)
