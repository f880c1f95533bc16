"""A Python model of a world state keyed by hashed keys, for checking the resident world state (phant_gpu_resident_state_*).

Roots come from the oracle's mptize (storage tries: keccak(slot) -> rlp(trim(value)); account trie: keccak(address) ->
rlp([nonce, balance, storageRoot, codeHash]), evmone mpt_hash.cpp:15-36).  Storage roots are cached per account and only
recomputed for accounts a diff touched."""
import numpy as np

from helpers import rlp_int_be, rlp_list, rlp_str
from oracle_lib import csr

DELETE, CLEAR = 1, 2
ZERO32 = bytes(32)


class Account:
    __slots__ = ("nonce", "balance", "code_hash", "storage", "sroot")

    def __init__(self):
        self.nonce, self.balance, self.code_hash, self.storage, self.sroot = 0, ZERO32, ZERO32, {}, None


class StateModel:
    def __init__(self, oracle):
        self.o = oracle
        self.acc = {}

    def copy(self):
        m = StateModel(self.o)
        for k, a in self.acc.items():
            b = Account()
            b.nonce, b.balance, b.code_hash, b.storage, b.sroot = a.nonce, a.balance, a.code_hash, dict(a.storage), a.sroot
            m.acc[k] = b
        return m

    def apply(self, d):
        """d: Diff.  Semantics of phant_gpu_resident_state_apply (include/phant_gpu.h)."""
        for key, flags, nonce, balance, code_hash in d.accounts:
            if flags & DELETE:
                self.acc.pop(key, None)
                continue
            a = self.acc.setdefault(key, Account())
            a.nonce, a.balance, a.code_hash = nonce, balance, code_hash
            if flags & CLEAR:
                a.storage, a.sroot = {}, None
        for ai, skey, val in d.slots:
            a = self.acc[d.accounts[ai][0]]
            if val == ZERO32:
                if a.storage.pop(skey, None) is not None:
                    a.sroot = None
            elif a.storage.get(skey) != val:
                a.storage[skey] = val
                a.sroot = None

    def storage_root(self, key):
        a = self.acc.get(key)
        if a is None:
            return ZERO32
        if a.sroot is None:
            ks = sorted(a.storage)
            keys = np.frombuffer(b"".join(ks), np.uint8) if ks else np.zeros(0, np.uint8)
            koff = np.arange(len(ks) + 1, dtype=np.uint32) * 32
            vals, voff = csr([rlp_str(a.storage[k].lstrip(b"\x00")) for k in ks], np.uint64)
            a.sroot = self.o.mptize_csr(keys, koff, vals, voff)
        return a.sroot

    def leaf(self, key):
        a = self.acc[key]
        return rlp_list([rlp_int_be(a.nonce.to_bytes(8, "big")), rlp_int_be(a.balance), rlp_str(self.storage_root(key)),
                         rlp_str(a.code_hash)])

    def root(self):
        ks = sorted(self.acc)
        keys = np.frombuffer(b"".join(ks), np.uint8) if ks else np.zeros(0, np.uint8)
        koff = np.arange(len(ks) + 1, dtype=np.uint32) * 32
        vals, voff = csr([self.leaf(k) for k in ks], np.uint64)
        return self.o.mptize_csr(keys, koff, vals, voff)


class Diff:
    """accounts: [(key32, flags, nonce, balance32, code_hash32)]; slots: [(account index, slot key32, value32)]"""

    def __init__(self, accounts=(), slots=()):
        self.accounts, self.slots = list(accounts), list(slots)

    def arrays(self):
        n, m = len(self.accounts), len(self.slots)
        cat = lambda xs: np.frombuffer(b"".join(xs), np.uint8).copy() if xs else np.zeros(0, np.uint8)  # noqa: E731
        return dict(account_keys32=cat([a[0] for a in self.accounts]), account_flags=np.array([a[1] for a in self.accounts], np.uint8),
                    nonce=np.array([a[2] for a in self.accounts], np.uint64), balance32=cat([a[3] for a in self.accounts]),
                    code_hash32=cat([a[4] for a in self.accounts]),
                    slot_account=np.array([s[0] for s in self.slots], np.uint32) if m else None,
                    slot_keys32=cat([s[1] for s in self.slots]) if m else None, slot_vals32=cat([s[2] for s in self.slots]) if m else None)


def hashed_table(keccak, table):
    """a fixture table (address / nonce / balance / code / storage, hex) -> {keccak(address): (nonce, balance32, codeHash,
    {keccak(slot): value32})}, zero slot values kept (they are writes of zero)"""
    out = {}
    for a in table:
        st = {keccak(bytes.fromhex(k)): bytes.fromhex(v).rjust(32, b"\x00") for k, v in a["storage"].items()}
        out[keccak(bytes.fromhex(a["address"]))] = (a["nonce"], bytes.fromhex(a["balance"]).rjust(32, b"\x00"),
                                                    keccak(bytes.fromhex(a["code"])), st)
    return out


def load_diff(h):
    """every account of a hashed table, with all its slots"""
    d = Diff()
    for k, (nonce, bal, ch, st) in h.items():
        d.accounts.append((k, 0, nonce, bal, ch))
        d.slots += [(len(d.accounts) - 1, sk, v) for sk, v in st.items()]
    return d


def change_diff(pre, post):
    """only what changed from hashed table `pre` to `post`: created, changed and destroyed accounts; changed and zeroed slots"""
    d = Diff()
    for k in pre:
        if k not in post:
            d.accounts.append((k, DELETE, 0, ZERO32, ZERO32))
    for k, (nonce, bal, ch, st) in post.items():
        old = pre.get(k)
        live = {sk: v for sk, v in st.items() if v != ZERO32}
        old_live = {} if old is None else {sk: v for sk, v in old[3].items() if v != ZERO32}
        changed = [(sk, v) for sk, v in live.items() if old_live.get(sk) != v] + [(sk, ZERO32) for sk in old_live if sk not in live]
        if old is not None and old[:3] == (nonce, bal, ch) and not changed:
            continue
        d.accounts.append((k, 0, nonce, bal, ch))
        d.slots += [(len(d.accounts) - 1, sk, v) for sk, v in changed]
    return d
