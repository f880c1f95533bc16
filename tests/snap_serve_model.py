"""The snap server's answers (phant_gpu_resident_state_snap_ranges: GetAccountRange and GetStorageRanges with byte budgets,
slim account bodies and boundary proofs) stated on the CPU, as go-ethereum's handler loops (ServiceGetAccountRangeQuery /
ServiceGetStorageRangesQuery) written in Python over the model state (tests/resident_state_model.py), with the proofs from
the C oracle's trie (oracle_trie_prove).  Also the consumer's side: slim bodies expanded to leaves, and each answer checked
with the CPU range-proof oracle (tests/range_proof_oracle.py) the way a syncing peer checks it.  TEST INFRASTRUCTURE."""
from helpers import EMPTY_ROOT, rlp_int_be, rlp_list, rlp_str
from range_proof_oracle import verify_range

EMPTY_CODE = bytes.fromhex("c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470")
ZERO = bytes(32)
FF = b"\xff" * 32


def slim(m, k):
    """account k's slim body: storageRoot and codeHash written as "" when they are the empty root and keccak("")"""
    a = m.acc[k]
    sroot = m.storage_root(k)
    return rlp_list([rlp_int_be(a.nonce.to_bytes(8, "big")), rlp_int_be(a.balance), rlp_str(b"" if sroot == EMPTY_ROOT else sroot),
                     rlp_str(b"" if a.code_hash == EMPTY_CODE else a.code_hash)])


def slot_body(v32):
    return rlp_str(bytes(v32).lstrip(b"\x00"))


def _items(b, pos, end):
    """the RLP items of b[pos:end] as (is_list, payload start, payload end); short forms and one-byte list lengths only, which
    is all a slim body uses"""
    out = []
    while pos < end:
        t = b[pos]
        if t < 0x80:
            out.append((False, pos, pos + 1))
        elif t <= 0xb7:
            out.append((False, pos + 1, pos + 1 + t - 0x80))
        elif t == 0xf8:
            out.append((True, pos + 2, pos + 2 + b[pos + 1]))
        elif t >= 0xc0:
            out.append((True, pos + 1, pos + 1 + t - 0xc0))
        else:
            raise ValueError("not a slim body")
        pos = out[-1][2]
    if pos != end:
        raise ValueError("not a slim body")
    return out


def full_leaf(body):
    """a slim body expanded to the account trie's leaf value: the empty storageRoot and codeHash put back"""
    (is_list, ps, pe), = _items(body, 0, len(body))
    f = [body[s:e] for lst, s, e in _items(body, ps, pe)]
    assert is_list and len(f) == 4
    return rlp_list([rlp_str(f[0]), rlp_str(f[1]), rlp_str(f[2] or EMPTY_ROOT), rlp_str(f[3] or EMPTY_CODE)])


class Prover:
    """oracle proof chains of the model's tries, built once per trie"""

    def __init__(self, oracle, m):
        self.o, self.m, self.tries = oracle, m, {}

    def chain(self, owner, key):
        if owner not in self.tries:
            if owner is None:
                kv = sorted((k, self.m.leaf(k)) for k in self.m.acc)
            else:
                a = self.m.acc.get(owner)
                kv = sorted((sk, slot_body(v)) for sk, v in a.storage.items()) if a else []
            self.tries[owner] = self.o.trie(kv) if kv else None
        t = self.tries[owner]
        return t.prove(key) if t is not None else []


def merge(first, last):
    """the wire list: the first chain's nodes, then the second's that are not already listed"""
    out = list(first)
    for x in last:
        if x not in out:
            out.append(x)
    return out


def account_answer(m, pv, origin, limit, nbytes):
    """-> ([(key, slim body)], proof)"""
    out, size = [], 0
    for k in sorted(m.acc):
        if k < origin:
            continue
        body = slim(m, k)
        out.append((k, body))
        size += 32 + len(body)
        if k >= limit or size > nbytes:
            break
    return out, merge(pv.chain(None, origin), pv.chain(None, out[-1][0]) if out else [])


def storage_answer(m, pv, accounts, origin, limit, nbytes):
    """-> ([[(key, body)] per served account], proof)"""
    hard = nbytes + nbytes // 10
    size, lists, proof = 0, [], []
    for i, acc in enumerate(accounts):
        if size >= nbytes:
            break
        o, lim = (origin, limit) if i == 0 else (ZERO, FF)
        a = m.acc.get(acc)
        lst, cut = [], False
        for k in sorted(a.storage) if a else []:
            if k < o:
                continue
            if size >= hard:
                cut = True
                break
            body = slot_body(a.storage[k])
            lst.append((k, body))
            size += 32 + len(body)
            if k >= lim:
                break
        lists.append(lst)
        if o != ZERO or (cut and lst):
            proof = merge(pv.chain(acc, o), pv.chain(acc, lst[-1][0]) if lst else [])
            break
    return lists, proof


def check_account_answer(keccak, root, origin, accounts, proof):
    """a syncing peer's check: (status, more) of the answer, slim bodies expanded"""
    return verify_range(keccak, proof, root, origin, [(k, full_leaf(b)) for k, b in accounts])


def check_storage_answer(keccak, m, accounts, origin, lists, proof):
    """every served list WHOLE against its storage root, except the last when a proof comes, checked from its origin"""
    out = []
    for i, lst in enumerate(lists):
        partial = bool(proof) and i + 1 == len(lists)
        a = accounts[i]
        sroot = m.storage_root(a) if a in m.acc else EMPTY_ROOT
        out.append(verify_range(keccak, proof if partial else [], sroot, origin if i == 0 else ZERO, lst, whole=not partial))
    return out
