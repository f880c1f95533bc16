"""Python host mirror of the reference functions on the hot path (names follow the Zig sources), over the
C ABI.  No arithmetic here -- flattening to CSR and one library call each.

  keccak256 / keccak256_with_prefix   src/crypto/hasher.zig:4-17
  KeyVal, mptize                      src/mpt/mpt.zig:13-45
  calculate_mpt_root                  src/blockchain/blockchain.zig:209-235
  payload_list_root                   src/engine_api/execution_payload.zig:125-139
  StateDB.root                        hook src/blockchain/blockchain.zig:83-85
  verify_witness                      hook src/engine_api/execution_payload.zig:177-178
  read_payload_witness                the pre-state StatelessPayloadStatusV1 (execution_payload.zig:20-25) needs first
"""
import numpy as np

from . import gpu

EMPTY_MPT_ROOT = bytes.fromhex("56e81f171bcc55a6ff8345e692c0f86e5b48e01b996cadc001622fb5e363b421")  # src/mpt/mpt.zig:10
EMPTY_CODE_HASH = bytes.fromhex("c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470")  # keccak("")


def _csr(items, dtype):
    off = np.zeros(len(items) + 1, dtype)
    if items:
        off[1:] = np.cumsum([len(x) for x in items])
    data = np.frombuffer(b"".join(bytes(x) for x in items) or b"\x00", np.uint8)
    return np.ascontiguousarray(data), off


def keccak256_batch(ctx, msgs):
    data, off = _csr(msgs, np.uint64)
    out = np.zeros((len(msgs), 32), np.uint8)
    ctx.keccak256_batch(data, off, len(msgs), out)
    return [o.tobytes() for o in out]


def keccak256(ctx, data):
    return keccak256_batch(ctx, [data])[0]


def keccak256_with_prefix(ctx, prefix, data):
    return keccak256(ctx, bytes(prefix) + bytes(data))


def tx_hashes(ctx, encoded_txs):
    """Tx.hash (src/types/transaction.zig:79-85) for a whole block: keccak256 of each encoded transaction
    (type byte || rlp for typed ones), one batched call (row N4 of SURVEY.md 8f: the hashing half of sender recovery)."""
    return keccak256_batch(ctx, encoded_txs)


def addresses_from_pubkeys(ctx, pubkeys65):
    """the last step of TxSigner.get_sender (src/signer/signer.zig:78): keccak256(pubkey[1..])[12..] for many
    public keys at once.  For keys that still have to be recovered use get_senders below: phant_gpu_ecrecover_batch fuses
    the secp256k1 recovery with this hashing step on the device, and get_senders does the `v` decoding and
    validateSignatureFields (ecdsa.zig:28-36) in front of it exactly as signer.zig:41-76 does."""
    return [h[12:] for h in keccak256_batch(ctx, [bytes(p)[1:] for p in pubkeys65])]


class KeyVal:
    """mpt.zig:13-34"""

    def __init__(self, key, value):
        self.nibbles = [n for b in bytes(key) for n in (b >> 4, b & 15)]
        self.value = bytes(value)

    init = classmethod(lambda cls, key, value: cls(key, value))

    @staticmethod
    def less_than(a, b):
        return a.nibbles < b.nibbles

    def key_bytes(self):
        return bytes((self.nibbles[i] << 4) | self.nibbles[i + 1] for i in range(0, len(self.nibbles), 2))


def mptize(ctx, keyvals):
    """mpt.zig:38-45; `keyvals` must be sorted by key (the reference asserts) -> PhantGpuError(-1) otherwise"""
    keys, koff = _csr([kv.key_bytes() for kv in keyvals], np.uint32)
    vals, voff = _csr([kv.value for kv in keyvals], np.uint64)
    return ctx.mpt_root(keys, koff, vals, voff, len(keyvals))


def mptize_many(ctx, lists):
    """many independent mptize calls as ONE forest build (phant_gpu_mpt_roots): lists = [[KeyVal, ...], ...]"""
    flat = [kv for lst in lists for kv in lst]
    keys, koff = _csr([kv.key_bytes() for kv in flat], np.uint32)
    vals, voff = _csr([kv.value for kv in flat], np.uint64)
    seg = np.zeros(len(lists) + 1, np.uint32)
    seg[1:] = np.cumsum([len(lst) for lst in lists])
    return ctx.mpt_roots(keys, koff, vals, voff, seg, len(lists))


def _index_keyvals(encoded_items):
    """blockchain.zig:214-232 key order"""
    n = len(encoded_items)
    kv, i = [], 0
    while i + 1 < n and i + 1 != 0x80:
        kv.append(KeyVal(bytes([i + 1]), encoded_items[i + 1]))
        i += 1
    if n > 0:
        kv.append(KeyVal(b"\x80", encoded_items[0]))
        i += 1
    while i < n:
        kv.append(KeyVal(_rlp_uint(i), encoded_items[i]))
        i += 1
    return kv


def calculate_mpt_roots(ctx, item_lists):
    """calculateMPTRoot for many lists at once (e.g. transactions / receipts / withdrawals of a range of blocks)"""
    return mptize_many(ctx, [_index_keyvals(items) for items in item_lists])


def _rlp_uint(i):
    if i == 0:
        return b"\x80"
    b = i.to_bytes((i.bit_length() + 7) // 8, "big")
    return b if len(b) == 1 and b[0] < 0x80 else bytes([0x80 + len(b)]) + b


def calculate_mpt_root(ctx, encoded_items):
    """blockchain.zig:209-235: keys rlp(index) visited in sorted order: 1..0x7f, then 0 (0x80), then 0x80.."""
    n = len(encoded_items)
    kv, i = [], 0
    while i + 1 < n and i + 1 != 0x80:
        kv.append(KeyVal(bytes([i + 1]), encoded_items[i + 1]))
        i += 1
    if n > 0:
        kv.append(KeyVal(b"\x80", encoded_items[0]))
        i += 1
    while i < n:
        kv.append(KeyVal(_rlp_uint(i), encoded_items[i]))
        i += 1
    return mptize(ctx, kv)


def payload_list_root(ctx, encoded_items):
    """execution_payload.zig:125-139: 32-byte big-endian index keys"""
    return mptize(ctx, [KeyVal(i.to_bytes(32, "big"), v) for i, v in enumerate(encoded_items)])


class AccountState:
    """src/state/types.zig:13-33"""

    def __init__(self, nonce=0, balance=0, code=b"", storage=None):
        self.nonce, self.balance, self.code, self.storage = nonce, balance, bytes(code), dict(storage or {})


class StateDB:
    """src/state/statedb.zig:16-30 (address -> AccountState) plus the root() the reference lacks"""

    def __init__(self):
        self.db = {}

    def root(self, ctx):
        accts = sorted(self.db.items())
        return ctx.state_root(len(accts), *_flatten_accounts(accts))

    # ---- the same root with the account trie sharded over GPUs by top nibble (SURVEY.md 8e) ----
    def hashed_top_nibbles(self, ctx):
        """(sorted account list, top nibble of keccak(address) per account): which root-branch slot each account is under"""
        accts = sorted(self.db.items())
        if not accts:
            return accts, np.zeros(0, np.uint8)
        h = keccak256_batch(ctx, [a for a, _ in accts])
        return accts, np.array([x[0] >> 4 for x in h], np.uint8)

    def local_subtree_roots(self, ctx, rank, world):
        """this rank's share: (16 x 32 subtree hashes, mask, accounts it holds) for the root-branch slots it owns"""
        from . import shard
        accts, nib = self.hashed_top_nibbles(ctx)
        mine = [accts[i] for i in range(len(accts)) if shard.nibble_owner(int(nib[i]), world) == rank]
        refs, mask = ctx.state_subtree_roots(len(mine), *_flatten_accounts(mine))
        return refs, mask, mine

    def root_sharded(self, ctx, rank, world, group=None):
        """StateDB.root() over `world` GPUs: every rank holds the same StateDB (phant's state lives on the host), builds the
        subtrees of its own top nibbles, ONE all-reduce of 16 x 32 bytes + presence flags, and every rank hashes the root
        branch itself.  Equals root() bit for bit."""
        from . import shard
        refs, mask, mine = self.local_subtree_roots(ctx, rank, world)
        refs_all, mask_all = shard.allgather_subtree_roots(refs, mask, group)
        if bin(mask_all).count("1") >= 2:
            return keccak256(ctx, shard.root_branch_rlp(refs_all, mask_all))
        # zero or one populated slot: the root is empty / a leaf / an extension, not a branch; the one rank that owns the
        # slot holds every account and computes the whole root, the others contribute zeros to a second 32-byte reduce
        full = np.zeros(32, np.uint8)
        if mask_all == 0:
            full = np.frombuffer(ctx.state_root(0, *_flatten_accounts([])), np.uint8).copy() if rank == 0 else full
        elif mask:
            full = np.frombuffer(ctx.state_root(len(mine), *_flatten_accounts(mine)), np.uint8).copy()
        return shard.sum_bytes(full, group).tobytes()


def _hashed_diff(ctx, touched, changed_slots, recreated):
    """ResidentStateDB.apply's arguments -> the keyword arrays of a phant_gpu_state_diff (addresses, slot numbers and code
    hashed with K); slot arrays are None when no slot is written"""
    from .gpu import ACCOUNT_CLEAR_STORAGE, ACCOUNT_DELETE
    addrs = list(touched)
    index = {a: i for i, a in enumerate(addrs)}
    recreated = set(recreated)
    if any(touched.get(a) is None for a in recreated):
        raise ValueError("a re-created account must be touched and live")
    flags = np.array([ACCOUNT_DELETE if touched[a] is None else
                      (ACCOUNT_CLEAR_STORAGE if changed_slots is None or a in recreated else 0) for a in addrs], np.uint8)
    slots = changed_slots if changed_slots is not None else {a: s.storage for a, s in touched.items() if s is not None}
    sa, sk, sv = [], [], []
    for a, writes in slots.items():
        if touched.get(a) is None:
            raise ValueError("slots of an account that is not touched and live")
        for k, v in writes.items():
            sa.append(index[a])
            sk.append(int(k).to_bytes(32, "big"))
            sv.append(int(v).to_bytes(32, "big"))
    live = [touched[a] or AccountState() for a in addrs]
    keys = np.frombuffer(b"".join(keccak256_batch(ctx, addrs)), np.uint8)
    code_hashes = np.frombuffer(b"".join(keccak256_batch(ctx, [s.code for s in live])), np.uint8)
    bal = np.frombuffer(b"".join(s.balance.to_bytes(32, "big") for s in live), np.uint8)
    nonce = np.array([s.nonce for s in live], np.uint64)
    d = dict(account_keys32=keys, nonce=nonce, balance32=bal, code_hash32=code_hashes, account_flags=flags, slot_account=None,
             slot_keys32=None, slot_vals32=None)
    if sa:
        d.update(slot_account=np.array(sa, np.uint32), slot_keys32=np.frombuffer(b"".join(keccak256_batch(ctx, sk)), np.uint8),
                 slot_vals32=np.frombuffer(b"".join(sv), np.uint8))
    return d


MAX_KEY = b"\xff" * 32  # the last hashed key: a range's limit when the caller wants to learn what follows
SNAP_SOFT_LIMIT = 2 << 20  # the most bytes a snap answer is asked to hold (go-ethereum's softResponseLimit)


def _next_key(k):
    """the hashed key after k (a range's next origin; k is never MAX_KEY when more follows it)"""
    return (int.from_bytes(k, "big") + 1).to_bytes(32, "big")


class ResidentStateDB:
    """StateDB.root() block after block with the world state resident on the device (gpu.ResidentState, DESIGN.md §4.3c):
    addresses, slot numbers and code are hashed with K, the diff is built from the touched accounts and the changed slots,
    and one apply returns the new root.  No storage root is computed on the host."""

    def __init__(self, ctx):
        self.ctx = ctx
        self.state = ctx.resident_state()
        self.journal = 0
        self.code_state = self.state  # the gpu.ResidentState whose code store put_codes, get_code and witness_blob use

    def set_journal(self, depth):
        """keep what undoes each of the last `depth` applies on the device, so that revert() can take blocks back"""
        self.state.set_journal(depth)
        self.journal = depth

    def revert(self, n=1):
        """undo the last n applies (a block whose root did not match its header, or the blocks a reorg leaves); returns the
        root before the oldest of them"""
        return self.state.revert(n)

    def fork(self, back=0):
        """a ResidentStateDB over a fork of this state (gpu.ResidentState.fork, DESIGN.md §4.3l): a new, independent state
        holding exactly what revert(back) would return to, while this one is not changed.  Every method works on it at that
        root: get_proofs, account_range_proof / storage_range_proof, get_trie_nodes, witness, read, dump, and apply for a
        side branch.  It starts with no journal.  Codes are addressed by hash, so the fork keeps using the code store of the
        state it was forked from (put_codes on the fork adds there): that state's prune_codes can drop codes only the fork
        still names, and the fork finds no code once that state is closed.  Close the fork when done."""
        db = ResidentStateDB.__new__(ResidentStateDB)
        db.ctx, db.state, db.journal, db.code_state = self.ctx, self.state.fork(back), 0, self.code_state
        return db

    def fork_at(self, root):
        """fork() at the `back` whose root is `root` (the root read(back) reports), or None when neither the current root
        nor any root the journal reaches is `root`.  The snap entry point: fork_at(pivot).get_trie_nodes(pivot, ...),
        .account_range_proof(...), .storage_range_proof(...) and .get_proofs(...) serve a syncing peer at its pivot while
        this state moves on."""
        root = bytes(root)
        none = np.zeros(0, np.uint8)
        for back in range(self.state.info()["journal_applies"] + 1):
            if (self.state.root() if back == 0 else self.state.read(none, back=back)[1]) == root:
                return self.fork(back)
        return None

    def load(self, statedb):
        """the first apply: every account of `statedb` with all its slots"""
        return self.apply(statedb.db)

    def apply(self, touched, changed_slots=None, recreated=()):
        """touched: address -> AccountState, or None for a destroyed account.  changed_slots: address -> {slot: new value}
        (0 = deleted) for the slots the block wrote, every address in it touched and live; None = send each touched
        account's whole storage in place of what the device holds (CLEAR_STORAGE).  recreated: addresses (touched, live)
        destroyed and created again in the block: their old storage is dropped before their changed slots apply.  apply
        does not need a codeHash's code to be held: put_codes(the block's new code) first to serve it with get_code and
        witness_blob."""
        addrs = list(touched)
        if not addrs:  # with a journal an empty block still counts as one apply, so that revert(k) undoes k blocks
            empty = np.zeros(0, np.uint8)
            return self.state.apply(empty, np.zeros(0, np.uint64), empty, empty) if self.journal else self.state.root()
        d = _hashed_diff(self.ctx, touched, changed_slots, recreated)
        if d["slot_account"] is None:
            return self.state.apply(d["account_keys32"], d["nonce"], d["balance32"], d["code_hash32"], d["account_flags"])
        return self.state.apply(**d)

    def witness(self, touched, changed_slots=None, recreated=()):
        """the execution witness of the block apply() would take with these arguments, from the state as it is now (which
        is not changed): the pre-state trie nodes the block reads or changes, each once, ordered by digest.  With the
        block's codes, encode_witness turns them into the blob transition_root reads (witness_blob does both)."""
        if not touched:
            return []
        d = _hashed_diff(self.ctx, touched, changed_slots, recreated)
        nodes, off = self.state.witness(**d)
        return [nodes[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]

    def put_codes(self, codes):
        """keep contract codes on the device beside the state, by keccak(code) (DESIGN.md §4.3i), for get_code, witness_blob
        and snap's GetByteCodes: put a block's new code before its apply, as load's caller puts the snapshot's.  A code
        already held is stored once; the empty code is never stored.  Returns the hashes, in order.  Codes stay until
        prune_codes() finds no reachable root that names them."""
        return [h.tobytes() for h in self.code_state.put_codes([bytes(c) for c in codes])]

    def prune_codes(self):
        """drop the held codes that no account names now or at any root revert() can return to"""
        self.code_state.prune_codes()

    def _code_hashes(self, addrs, back):
        """each address's codeHash at that root: keccak("") for an absent account"""
        akeys = np.frombuffer(b"".join(keccak256_batch(self.ctx, addrs)), np.uint8)
        r, _ = self.state.read(akeys, back=back)
        return [r["code_hash32"][i].tobytes() if r["account_status"][i] == 1 else EMPTY_CODE_HASH for i in range(len(addrs))]

    def get_code(self, addresses, back=0):
        """eth_getCode for many addresses at the state as it is now (back = 0) or `back` applies ago: read's codeHash, then one
        lookup in the code store.  Returns address -> code bytes: b"" for an absent account or an account without code, None
        when the store does not hold the code its codeHash names."""
        addrs = list(dict.fromkeys(bytes(a) for a in addresses))
        if not addrs:
            return {}
        status, codes = self.code_state.codes(np.frombuffer(b"".join(self._code_hashes(addrs, back)), np.uint8))
        return {a: codes[i] if status[i] == 1 else None for i, a in enumerate(addrs)}

    def witness_blob(self, touched, changed_slots=None, recreated=(), headers=()):
        """the whole execution witness of the block apply() would take with these arguments, as read_payload_witness and
        transition_root read it: encode_witness(headers, codes, witness(...)).  codes are the distinct codes of every listed
        account present before the block with code, ordered by hash, from the code store.  Raises ValueError naming the
        addresses whose code the store does not hold: a witness without them could not be executed."""
        nodes = self.witness(touched, changed_slots, recreated)
        addrs = [bytes(a) for a in touched]
        by_hash = {}
        for a, h in zip(addrs, self._code_hashes(addrs, 0) if addrs else []):
            if h != EMPTY_CODE_HASH:
                by_hash.setdefault(h, []).append(a)
        hashes = sorted(by_hash)
        codes = []
        if hashes:
            status, codes = self.code_state.codes(np.frombuffer(b"".join(hashes), np.uint8))
            missing = [a for i, h in enumerate(hashes) if status[i] != 1 for a in by_hash[h]]
            if missing:
                raise ValueError("the code store does not hold the code of " + ", ".join("0x" + a.hex() for a in missing))
        return encode_witness(headers, codes, nodes)

    def get_proofs(self, requests):
        """eth_getProof (EIP-1186) under the state as it is now (which is not changed), for many addresses in one call.
        requests: address -> [slot number, ...].  Returns address -> {accountProof, nonce, balance, storageHash, codeHash,
        storageProof: [{key, value, proof}]}, each proof a list of node bytes, root first.  An absent account gets the fields
        of an empty account -- nonce 0, balance 0, the empty trie root and keccak("") -- with a proof of its absence, and its
        slots value 0 with empty proofs (they hang from the empty root).  An absent slot has value 0 and a proof of its absence."""
        addrs = list(requests)
        if not addrs:
            return {}
        slots = [(i, int(s)) for i, a in enumerate(addrs) for s in requests[a]]
        akeys = np.frombuffer(b"".join(keccak256_batch(self.ctx, addrs)), np.uint8)
        sa = np.array([i for i, _ in slots], np.uint32) if slots else None
        sk = np.frombuffer(b"".join(keccak256_batch(self.ctx, [s.to_bytes(32, "big") for _, s in slots])), np.uint8) if slots else None
        r = self.state.prove(akeys, sa, sk)
        nodes, off, idx, first = r["nodes"], r["node_off"], r["node_index"], r["proof_first"]
        node = lambda k: nodes[int(off[k]):int(off[k + 1])].tobytes()  # noqa: E731
        chain = lambda p: [node(int(k)) for k in idx[int(first[p]):int(first[p + 1])]]  # noqa: E731
        out = {}
        for i, a in enumerate(addrs):
            present = r["status"][i] == 1
            out[a] = dict(accountProof=chain(i), nonce=int(r["nonce"][i]), balance=int.from_bytes(r["balance32"][i].tobytes(), "big"),
                          storageHash=r["storage_root32"][i].tobytes() if present else EMPTY_MPT_ROOT,
                          codeHash=r["code_hash32"][i].tobytes() if present else EMPTY_CODE_HASH, storageProof=[])
        for j, (i, s) in enumerate(slots):
            out[addrs[i]]["storageProof"].append(dict(key=s, value=int.from_bytes(r["slot_vals32"][j].tobytes(), "big"),
                                                      proof=chain(len(addrs) + j)))
        return out

    def read(self, requests, back=0):
        """eth_getBalance / eth_getTransactionCount / eth_getStorageAt (and the codeHash behind eth_getCode) for many
        addresses in one call, with no proof and no hashing of trie nodes: at the state as it is now (back = 0) or as it was
        `back` applies ago (1 <= back <= the journal's applies), which is not changed.  requests: address -> [slot number, ...].
        Returns address -> {nonce, balance, storageHash, codeHash, exists, storage: {slot: value}}; an absent account gets the
        fields of an empty account -- nonce 0, balance 0, the empty trie root and keccak("") -- and value 0 for its slots."""
        addrs = list(requests)
        if not addrs:
            return {}
        slots = [(i, int(s)) for i, a in enumerate(addrs) for s in requests[a]]
        akeys = np.frombuffer(b"".join(keccak256_batch(self.ctx, addrs)), np.uint8)
        sa = np.array([i for i, _ in slots], np.uint32) if slots else None
        sk = np.frombuffer(b"".join(keccak256_batch(self.ctx, [s.to_bytes(32, "big") for _, s in slots])), np.uint8) if slots else None
        r, _ = self.state.read(akeys, sa, sk, back=back)
        out = {}
        for i, a in enumerate(addrs):
            present = r["account_status"][i] == 1
            out[a] = dict(nonce=int(r["nonce"][i]), balance=int.from_bytes(r["balance32"][i].tobytes(), "big"),
                          storageHash=r["storage_root32"][i].tobytes() if present else EMPTY_MPT_ROOT,
                          codeHash=r["code_hash32"][i].tobytes() if present else EMPTY_CODE_HASH, exists=bool(present), storage={})
        for j, (i, s) in enumerate(slots):
            out[addrs[i]]["storage"][s] = int.from_bytes(r["slot_vals32"][j].tobytes(), "big")
        return out

    @staticmethod
    def _accounts(r, a, b):
        return [(r["account_keys32"][e].tobytes(), dict(nonce=int(r["nonce"][e]), balance=int.from_bytes(r["balance32"][e].tobytes(), "big"),
                                                        storageHash=r["storage_root32"][e].tobytes(), codeHash=r["code_hash32"][e].tobytes()))
                for e in range(a, b)]

    @staticmethod
    def _slots(r, a, b):
        return [(r["slot_keys32"][e].tobytes(), int.from_bytes(r["slot_vals32"][e].tobytes(), "big")) for e in range(a, b)]

    def account_range(self, origin, limit=MAX_KEY, max_entries=256, back=0):
        """debug_accountRange / snap GetAccountRange without proofs: the first `max_entries` accounts whose hashed key lies in
        [origin, limit] (32-byte keys, inclusive), ascending, at the state as it is now (back = 0) or `back` applies ago,
        which is not changed.  Returns ([(hashed key, {nonce, balance, storageHash, codeHash})], more): more is True when
        the range holds further accounts.  Keys are hashed: the state holds no preimages."""
        r, _ = self.state.range([(origin, limit, max_entries)], back=back)
        return self._accounts(r, 0, int(r["account_first"][1])), bool(r["account_more"][0])

    def storage_range(self, address, origin, limit=MAX_KEY, max_entries=256, back=0):
        """debug_storageRangeAt / snap GetStorageRanges without proofs: the first `max_entries` slots of `address` whose
        hashed slot key lies in [origin, limit], ascending, at the state now or `back` applies ago.  Returns ([(hashed slot
        key, value)], more); an account absent at that root has no slots."""
        akey = keccak256_batch(self.ctx, [address])[0]
        r, _ = self.state.range(storage_ranges=[(akey, origin, limit, max_entries)], back=back)
        return self._slots(r, 0, int(r["slot_first"][1])), bool(r["slot_more"][0])

    def dump(self, back=0, chunk=1 << 20):
        """the whole state now or `back` applies ago, read in calls of at most `chunk` entries: the accounts range by range,
        then the slots of every account whose storageRoot is not the empty root, many accounts per call.  Returns {hashed
        address: (nonce, balance32, codeHash, {hashed slot: value32})}."""
        out, rich, origin = {}, [], bytes(32)
        while True:
            r, _ = self.state.range([(origin, MAX_KEY, chunk)], back=back)
            for k, a in self._accounts(r, 0, int(r["account_first"][1])):
                out[k] = (a["nonce"], a["balance"].to_bytes(32, "big"), a["codeHash"], {})
                if a["storageHash"] != EMPTY_MPT_ROOT:
                    rich.append(k)
            if not r["account_more"][0]:
                break
            origin = _next_key(k)
        pending = [(k, bytes(32)) for k in rich]  # (account, next origin)
        while pending:
            batch = pending[:chunk]
            each = max(chunk // len(batch), 1)
            r, _ = self.state.range(storage_ranges=[(k, o, MAX_KEY, each) for k, o in batch], back=back)
            first = r["slot_first"]
            pending = pending[len(batch):]
            for i, (k, _) in enumerate(batch):
                slots = self._slots(r, int(first[i]), int(first[i + 1]))
                out[k][3].update((sk, v.to_bytes(32, "big")) for sk, v in slots)
                if r["slot_more"][i]:
                    pending.append((k, _next_key(slots[-1][0])))
        return out

    def account_range_proof(self, origin, limit=MAX_KEY, max_entries=256):
        """snap GetAccountRange at the current root: account_range() plus the boundary proofs, one prove() call on the origin
        and the last key returned (once when they are the same key).  Returns dict(accounts, more, keys (the proven keys:
        origin first), proof (gpu.ResidentState.prove's batch))."""
        accounts, more = self.account_range(origin, limit, max_entries)
        keys = list(dict.fromkeys([origin] + ([accounts[-1][0]] if accounts else [])))
        return dict(accounts=accounts, more=more, keys=keys, proof=self.state.prove(np.frombuffer(b"".join(keys), np.uint8)))

    def storage_range_proof(self, address, origin, limit=MAX_KEY, max_entries=256):
        """snap GetStorageRanges for one account at the current root: storage_range() plus the boundary proofs in the
        account's storage trie (proof 0 is the account's own, then one per proven slot key: origin first, the last slot
        returned second unless it is the origin)."""
        slots, more = self.storage_range(address, origin, limit, max_entries)
        keys = list(dict.fromkeys([origin] + ([slots[-1][0]] if slots else [])))
        akey = keccak256_batch(self.ctx, [address])[0]
        proof = self.state.prove(np.frombuffer(akey, np.uint8), np.zeros(len(keys), np.uint32), np.frombuffer(b"".join(keys), np.uint8))
        return dict(slots=slots, more=more, keys=keys, proof=proof)

    def get_trie_nodes(self, root, pathsets, max_bytes=2 << 20):
        """snap GetTrieNodes at the current root, for a healing peer: pathsets as the wire carries them -- [path] for a node of
        the account trie, [account hash (32 bytes), path, ...] for nodes of that account's storage trie -- each path
        compact-encoded (hex-prefix with flag nibble 0 for an even, 1 for an odd number of nibbles).  Returns one blob per path
        in request order: the node's RLP (the root, or a node its parent references by hash), b"" when there is no such node
        or the path does not decode.  It stops after the blob that takes the running total past max_bytes, and returns []
        when `root` is not the current root (past roots are not served)."""
        if bytes(root) != self.state.root():
            return []
        owners, slot, paths, lens, tries = {}, [], [], [], []  # slot[i]: index of path i in the device request, or None
        for ps in pathsets:
            ps = [bytes(x) for x in ps]
            if not ps:
                continue
            if len(ps) == 1:
                trie, rest = 0, ps
            else:
                trie, rest = (1 + owners.setdefault(ps[0], len(owners)) if len(ps[0]) == 32 else None), ps[1:]
            for c in rest:
                p = _compact_path(c) if trie is not None else None
                slot.append(None if p is None else len(paths))
                if p is not None:
                    paths.append(p[0]); lens.append(p[1]); tries.append(trie)
        status, blobs = [], []
        if paths:
            status, blobs = self.state.trie_nodes(np.frombuffer(b"".join(paths), np.uint8), np.array(lens, np.uint8),
                                                  np.array(tries, np.uint32),
                                                  np.frombuffer(b"".join(owners), np.uint8) if owners else None)
        out, total = [], 0
        for j in slot:
            b = blobs[j] if j is not None and status[j] == 1 else b""
            out.append(b)
            total += len(b)
            if total > max_bytes:
                break
        return out

    def snap_account_range(self, root, origin, limit=MAX_KEY, nbytes=SNAP_SOFT_LIMIT):
        """snap GetAccountRange at the current root, as a snap server answers it (DESIGN.md §4.3m): the accounts from
        `origin` ascending, up to and including the first at or past `limit`, until their wire size passes nbytes (capped at
        2 MiB; at least one account when any follows origin).  Returns (accounts=[(hashed key, slim body)], proof=[node
        bytes]): the origin's proof, then the last account's nodes not already listed.  An empty answer when `root` is not
        the current root: serve a pivot through fork_at(root)."""
        ans = self.serve_snap([(root, origin, limit, nbytes)])[0]
        return ans if ans is not None else ([], [])

    def snap_storage_ranges(self, root, accounts, origin=bytes(32), limit=MAX_KEY, nbytes=SNAP_SOFT_LIMIT):
        """snap GetStorageRanges at the current root: accounts are hashed account keys; origin and limit apply to the first
        of them.  Returns (slots=[[(hashed slot, body)] per served account], proof=[node bytes]); the proof, when there is
        one, is the last served account's, and that account's answer is partial.  An empty answer when `root` is not the
        current root."""
        ans = self.serve_snap([(root, list(accounts), origin, limit, nbytes)])[0]
        return ans if ans is not None else ([], [])

    def serve_snap(self, requests):
        """many peers' GetAccountRange and GetStorageRanges requests answered in one device call: each request is (root,
        origin, limit, nbytes) for an account range or (root, [hashed accounts], origin, limit, nbytes) for storage ranges.
        Returns one (entries, proof) per request in order, as snap_account_range / snap_storage_ranges return them, or None
        for a request whose root is not the current root.  Budgets are capped at 2 MiB."""
        cur = self.state.root()
        ar, sr, where = [], [], []
        for r in requests:
            if bytes(r[0]) != cur:
                where.append(None)
            elif len(r) == 4:
                where.append((0, len(ar)))
                ar.append((bytes(r[1]), bytes(r[2]), min(int(r[3]), SNAP_SOFT_LIMIT)))
            else:
                where.append((1, len(sr)))
                sr.append(([bytes(a) for a in r[1]], bytes(r[2]), bytes(r[3]), min(int(r[4]), SNAP_SOFT_LIMIT)))
        if not ar and not sr:
            return [None] * len(requests)
        a = self.state.snap_ranges(ar, sr)
        out = []
        for w in where:
            if w is None:
                out.append(None)
            elif w[0] == 0:
                out.append((a["accounts"][w[1]], a["proofs"][w[1]]))
            else:
                out.append((a["slots"][w[1]], a["proofs"][len(ar) + w[1]]))
        return out

    def close(self):
        self.state.close()


def _compact_path(b):
    """a compact-encoded trie path (hex-prefix, flag nibble 0: even, 1: odd) -> (its nibbles packed high nibble first and
    padded to 32 bytes, nibble count); None when it does not decode as one or holds more than 64 nibbles"""
    if not b or b[0] >> 4 > 1 or (b[0] >> 4 == 0 and b[0] & 15):
        return None
    nib = ([b[0] & 15] if b[0] >> 4 else []) + [x for c in b[1:] for x in (c >> 4, c & 15)]
    if len(nib) > 64:
        return None
    packed = bytes((nib[i] << 4) | (nib[i + 1] if i + 1 < len(nib) else 0) for i in range(0, len(nib), 2))
    return packed.ljust(32, b"\x00"), len(nib)


def _flatten_accounts(accts):
    """[(address, AccountState)] -> the SoA / CSR tables of phant_gpu_accounts (include/phant_gpu.h)"""
    n = len(accts)
    one = np.zeros(1, np.uint8)
    addr = np.frombuffer(b"".join(a for a, _ in accts), np.uint8) if n else one
    nonce = np.array([s.nonce for _, s in accts], np.uint64) if n else np.zeros(1, np.uint64)
    bal = np.frombuffer(b"".join(s.balance.to_bytes(32, "big") for _, s in accts), np.uint8) if n else one
    code, coff = _csr([s.code for _, s in accts], np.uint64)
    sk, sv, soff = [], [], [0]
    for _, s in accts:
        for k, v in s.storage.items():
            sk.append(int(k).to_bytes(32, "big"))
            sv.append(int(v).to_bytes(32, "big"))
        soff.append(len(sk))
    skeys = np.frombuffer(b"".join(sk), np.uint8) if sk else one
    svals = np.frombuffer(b"".join(sv), np.uint8) if sv else one
    return addr, nonce, bal, code, coff, skeys, svals, np.array(soff, np.uint64)


def run_block_post_checks(ctx, header, encoded_txs, encoded_receipts, encoded_withdrawals, statedb=None):
    """The root comparisons at the end of Blockchain.runBlock (src/blockchain/blockchain.zig:76-90), all tries of the block
    in ONE forest build.  `header` is a dict with transactions_root / receipts_root / withdrawals_root (/ state_root).
    Returns the list of mismatching field names (empty = block passes).  The state-root comparison is the one phant has
    commented out (:83-85); it runs when a StateDB is given."""
    lists = [encoded_txs, encoded_withdrawals] + ([encoded_receipts] if encoded_receipts is not None else [])
    roots = calculate_mpt_roots(ctx, lists)
    bad = []
    if roots[0] != header["transactions_root"]:
        bad.append("transactions_root")
    if roots[1] != header["withdrawals_root"]:
        bad.append("withdrawals_root")
    if encoded_receipts is not None and roots[2] != header["receipts_root"]:
        bad.append("receipts_root")
    if statedb is not None and statedb.root(ctx) != header["state_root"]:
        bad.append("state_root")
    return bad


class Log:
    """src/types/receipt.zig:65-69"""

    def __init__(self, address, topics, data=b""):
        self.address, self.topics, self.data = bytes(address), [bytes(t) for t in topics], bytes(data)


def calculate_logs_blooms(ctx, receipts_logs):
    """Receipt.calculateLogsBloom (src/types/receipt.zig:37-48) for a whole block: receipts_logs = one list of Log per
    receipt -> (list of 256-byte blooms, block bloom = their OR, the check disabled at src/blockchain/blockchain.zig:86-88)"""
    items, owner = [], []
    for r, logs in enumerate(receipts_logs):
        for log in logs:
            items.append(log.address)
            owner.append(r)
            for t in log.topics:
                items.append(t)
                owner.append(r)
    n = len(receipts_logs)
    blooms = np.zeros((max(n, 1), 256), np.uint8)
    if n:
        data, off = _csr(items, np.uint64)
        ctx.logs_bloom(data, off, np.array(owner or [0], np.uint32), len(items), n, blooms)
    block = np.bitwise_or.reduce(blooms[:n], axis=0) if n else np.zeros(256, np.uint8)
    return [b.tobytes() for b in blooms[:n]], block.tobytes()


def _rlp_str(b):
    b = bytes(b)
    if len(b) == 1 and b[0] < 0x80:
        return b
    if len(b) <= 55:
        return bytes([0x80 + len(b)]) + b
    ll = (len(b).bit_length() + 7) // 8
    return bytes([0xb7 + ll]) + len(b).to_bytes(ll, "big") + b


def _rlp_list(items):
    body = b"".join(items)
    if len(body) <= 55:
        return bytes([0xc0 + len(body)]) + body
    ll = (len(body).bit_length() + 7) // 8
    return bytes([0xf7 + ll]) + len(body).to_bytes(ll, "big") + body


class Receipt:
    """src/types/receipt.zig:13-35: succeeded, cumulative_gas_used, bloom, logs.  `tx_type` (0 legacy) adds the EIP-2718
    type byte in front of the RLP, which phant's struct does not carry yet (its receipts root only matches legacy blocks)."""

    def __init__(self, succeeded, cumulative_gas_used, logs, tx_type=0):
        self.succeeded, self.cumulative_gas_used, self.logs, self.tx_type = bool(succeeded), int(cumulative_gas_used), list(logs), tx_type
        self.bloom = bytes(256)

    def encode(self):
        """Receipt.encode (receipt.zig:29-35): rlp([succeeded, cumulative_gas_used, bloom, logs])"""
        gas = self.cumulative_gas_used.to_bytes(8, "big").lstrip(b"\x00")
        logs = _rlp_list([_rlp_list([_rlp_str(l.address), _rlp_list([_rlp_str(t) for t in l.topics]), _rlp_str(l.data)]) for l in self.logs])
        body = _rlp_list([_rlp_str(b"\x01" if self.succeeded else b""), _rlp_str(gas), _rlp_str(self.bloom), logs])
        return (bytes([self.tx_type]) if self.tx_type else b"") + body


def receipts_root(ctx, receipts):
    """blockchain.zig:184-203: blooms of all receipts in one batched call (GPU), encodings on the host, receipts trie on
    the GPU.  Returns (receipts_root, block logs bloom)."""
    blooms, block_bloom = calculate_logs_blooms(ctx, [r.logs for r in receipts])
    for r, b in zip(receipts, blooms):
        r.bloom = b
    return calculate_mpt_root(ctx, [r.encode() for r in receipts]), block_bloom


def verify_witness_nodes(ctx, state_root, nodes, hashed_keys):
    """execution_payload.zig:177-178 for a witness that is an unordered SET of trie nodes (`state: [node, ...]`):
    -> status per key: 0 reject, 1 present, 2 absent, 3 node missing from the set"""
    n = len(hashed_keys)
    if n == 0:
        return []
    data, off = _csr(list(nodes), np.uint64)
    keys = np.frombuffer(b"".join(hashed_keys), np.uint8)
    status = np.zeros(n, np.uint8)
    ctx.verify_witness(len(nodes), data, off, n, keys, np.frombuffer(bytes(state_root), np.uint8), 1, None, status, None, None)
    return status.tolist()


def verify_witness(ctx, state_root, proofs):
    """proofs: list of (hashed_key32, [node bytes, root first]).  Returns the status list (0 reject / 1 present /
    2 absent); execution_payload.zig:177-178 would refuse the payload unless none is 0."""
    n = len(proofs)
    if n == 0:
        return []
    nodes, node_off = _csr([nd for _, chain in proofs for nd in chain], np.uint64)
    first = np.zeros(n + 1, np.uint64)
    first[1:] = np.cumsum([len(chain) for _, chain in proofs])
    keys = np.frombuffer(b"".join(k for k, _ in proofs), np.uint8)
    root = np.frombuffer(bytes(state_root), np.uint8)
    status = np.zeros(n, np.uint8)
    bitmap = np.zeros((n + 63) // 64, np.uint64)
    ctx.verify_proofs(n, nodes, node_off, first, keys, root, 1, bitmap, status, None, None)
    return status.tolist()


# ---- the witness wire format (SURVEY.md 8f N2) ------------------------------------------------------------------------------
# The reference carries the witness as an opaque byte string whose layout it leaves undefined
# (src/engine_api/execution_payload.zig:20-34 `witness: []const u8`, TODO at :177-178).  This mirror reads the layout geth's
# stateless mode puts on the wire -- rlp([headers, codes, state]), `state` the unordered set of trie nodes -- with strict,
# canonical RLP (the same rules the proof walk applies to nodes); anything else raises InvalidWitness.
class InvalidWitness(ValueError):
    pass


def _rlp_header(b, pos, end):
    """(is_list, payload_start, payload_end) of the item at pos; canonical encodings only"""
    if pos >= end:
        raise InvalidWitness("truncated item")
    t = b[pos]
    if t < 0x80:
        return False, pos, pos + 1
    short, long_ = (0x80, 0xb7) if t < 0xc0 else (0xc0, 0xf7)
    if t <= long_:
        start, ln = pos + 1, t - short
        if short == 0x80 and ln == 1 and start < end and b[start] < 0x80:
            raise InvalidWitness("single byte below 0x80 must encode itself")
    else:
        ll = t - long_
        if pos + 1 + ll > end or b[pos + 1] == 0:
            raise InvalidWitness("bad length of length")
        ln = int.from_bytes(b[pos + 1:pos + 1 + ll], "big")
        if ln < 56:
            raise InvalidWitness("long form used for a short payload")
        start = pos + 1 + ll
    if start + ln > end:
        raise InvalidWitness("item overruns its container")
    return t >= 0xc0, start, start + ln


def _rlp_list_items(b, start, end):
    pos, out = start, []
    while pos < end:
        is_list, ps, pe = _rlp_header(b, pos, end)
        out.append((is_list, pos, ps, pe))
        pos = pe
    return out


def decode_witness(blob):
    """witness bytes -> (headers: [raw rlp], codes: [bytes], nodes: [bytes]); raises InvalidWitness"""
    b = bytes(blob)
    is_list, ps, pe = _rlp_header(b, 0, len(b))
    if not is_list or pe != len(b):
        raise InvalidWitness("witness is not one RLP list")
    fields = _rlp_list_items(b, ps, pe)
    if len(fields) != 3 or not all(f[0] for f in fields):
        raise InvalidWitness("witness must be [headers, codes, state]")
    headers = []
    for is_l, p0, _, e in _rlp_list_items(b, fields[0][2], fields[0][3]):
        if not is_l:
            raise InvalidWitness("header is not a list")
        headers.append(b[p0:e])
    out = []
    for f in fields[1:]:
        items = _rlp_list_items(b, f[2], f[3])
        if any(it[0] for it in items):
            raise InvalidWitness("code / node is not a byte string")
        out.append([b[s:e] for _, _, s, e in items])
    return headers, out[0], out[1]


def encode_witness(headers, codes, nodes):
    """inverse of decode_witness (headers already RLP-encoded)"""
    return _rlp_list([_rlp_list(list(headers)), _rlp_list([_rlp_str(c) for c in codes]), _rlp_list([_rlp_str(n) for n in nodes])])


def verify_payload_witness(ctx, state_root, witness_blob, hashed_keys):
    """What newPayloadV2Handler's TODO (execution_payload.zig:177-178) asks for: decode the payload's witness and check that
    every touched key resolves inside its node set from `state_root`.  Returns the per-key status list; raises
    InvalidWitness for an undecodable blob.  The payload is refused unless every status is 1 or 2."""
    _, _, nodes = decode_witness(witness_blob)
    return verify_witness_nodes(ctx, state_root, nodes, hashed_keys)


class PreState:
    """What an execution witness proves about the state a block reads (read_payload_witness):
      accounts       address -> AccountState (src/state/types.zig:13-33) for every account the witness proves present, its
                     `storage` holding the requested slots proven non-zero (a slot proven absent is zero and is not stored);
      account_status address -> 0 reject / 1 present / 2 absent / 3 node missing;
      slot_status    (address, slot) -> the same four values;
      missing_code   addresses whose codeHash no code of the witness hashes to (their AccountState.code stays empty)."""

    def __init__(self):
        self.accounts, self.account_status, self.slot_status, self.missing_code = {}, {}, {}, []

    @property
    def complete(self):
        """every read proven (present or absent) and every present account's code supplied: the block can be executed"""
        return (all(s in (1, 2) for s in self.account_status.values()) and all(s in (1, 2) for s in self.slot_status.values())
                and not self.missing_code)

    def statedb(self):
        db = StateDB()
        db.db = dict(self.accounts)
        return db


def read_payload_witness(ctx, state_root, witness_blob, addresses, slots=()):
    """The pre-state a stateless client loads before it executes a block: the witness blob decoded, the addresses and slot
    numbers hashed (one K call each), then ONE pre-state read (phant_gpu_read_state): every account walked from `state_root`
    and decoded, every slot walked from its account's proven storage root, codes matched by hash -- all on the device.
    addresses: 20-byte addresses; slots: (address, slot number) pairs, the address need not be listed in `addresses`.
    Returns a PreState; raises InvalidWitness for an undecodable blob."""
    _, codes, nodes = decode_witness(witness_blob)
    addrs = list(dict.fromkeys([bytes(a) for a in addresses] + [bytes(a) for a, _ in slots]))
    out = PreState()
    if not addrs:
        return out
    idx = {a: i for i, a in enumerate(addrs)}
    na, ns = len(addrs), len(slots)
    akeys = np.frombuffer(b"".join(keccak256_batch(ctx, addrs)), np.uint8)
    skeys = np.frombuffer(b"".join(keccak256_batch(ctx, [int(s).to_bytes(32, "big") for _, s in slots])), np.uint8) if ns else None
    sacc = np.array([idx[bytes(a)] for a, _ in slots], np.uint32) if ns else None
    ndata, noff = _csr(list(nodes), np.uint64)
    cdata, coff = _csr(list(codes), np.uint64)
    st, nonce = np.zeros(na, np.uint8), np.zeros(na, np.uint64)
    bal, cidx = np.zeros((na, 32), np.uint8), np.zeros(na, np.uint32)
    sst, svals = np.zeros(max(ns, 1), np.uint8), np.zeros((max(ns, 1), 32), np.uint8)
    ctx.read_state(len(nodes), ndata, noff, na, akeys, np.frombuffer(bytes(state_root), np.uint8), 1, ns, skeys, sacc, len(codes), cdata, coff,
                   account_status=st, nonce=nonce, balance32=bal, code_index=cidx, slot_status=sst if ns else None,
                   slot_vals32=svals if ns else None)
    for i, a in enumerate(addrs):
        out.account_status[a] = int(st[i])
        if st[i] != 1:
            continue
        code = b""
        if cidx[i] == gpu.CODE_MISSING:
            out.missing_code.append(a)
        elif cidx[i] != gpu.CODE_EMPTY:
            code = bytes(codes[int(cidx[i])])
        out.accounts[a] = AccountState(int(nonce[i]), int.from_bytes(bal[i].tobytes(), "big"), code)
    for j, (a, s) in enumerate(slots):
        a = bytes(a)
        out.slot_status[(a, int(s))] = int(sst[j])
        v = int.from_bytes(svals[j].tobytes(), "big")
        if sst[j] == 1 and a in out.accounts:
            out.accounts[a].storage[int(s)] = v
    return out


# ---- transaction senders (SURVEY.md 8f N4): TxSigner.get_sender for a whole block -------------------------------------------
SECP256K1_N = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141
SPEC_TEST_CHAIN_ID = 0  # src/config/config.zig:9: legacy transactions are hashed without the EIP-155 fields on this chain


class SenderError(ValueError):
    """the error names of the reference: InvalidR / InvalidS (src/crypto/ecdsa.zig:28-36), EIP155_v (src/signer/signer.zig:59),
    InvalidTransaction (undecodable), RecoveryFailed (libsecp256k1 recovers no key)"""


def _tx_signing_parts(encoded, chain_id):
    """one encoded transaction -> (bytes whose keccak256 is the signing hash, r, s, recid); follows TxSigner.get_sender and
    hashTx (src/signer/signer.zig:41-188).  The unsigned fields are taken as the raw RLP items of the encoded transaction:
    for a canonical encoding that is byte-identical to re-serialising the decoded fields, which is what the reference does."""
    b = bytes(encoded)
    try:
        typed = len(b) > 0 and b[0] in (1, 2)
        body = b[1:] if typed else b
        is_list, ps, pe = _rlp_header(body, 0, len(body))
        if not is_list or pe != len(body):
            raise InvalidWitness("not one list")
        items = _rlp_list_items(body, ps, pe)
    except InvalidWitness as e:
        raise SenderError("InvalidTransaction") from e
    want = {False: 9, True: 11 if b[:1] == b"\x01" else 12}[typed]
    if len(items) != want or any(it[0] for it in items[-3:]):
        raise SenderError("InvalidTransaction")
    v, r, s = (int.from_bytes(body[it[2]:it[3]], "big") for it in items[-3:])
    if r > SECP256K1_N:                 # ecdsa.zig:29 (r == n passes here and fails in the recovery, as in the reference)
        raise SenderError("InvalidR")
    if s > SECP256K1_N // 2:            # ecdsa.zig:33: malleability rule
        raise SenderError("InvalidS")
    raw = [body[it[1]:it[3]] for it in items[:-3]]
    if typed:
        if v > 1:
            raise SenderError("InvalidTransaction")  # y_parity is one bit
        return b[:1] + _rlp_list(raw), r, s, v
    if v in (27, 28):
        recid = v - 27
    else:
        v155 = 35 + 2 * chain_id
        if v not in (v155, v155 + 1):
            raise SenderError("EIP155_v")
        recid = v - v155
    if chain_id != SPEC_TEST_CHAIN_ID:   # signer.zig:87: EIP-155 form whenever the signer's chain is not the spec-test chain
        raw = raw + [_rlp_uint(chain_id), b"\x80", b"\x80"]
    return _rlp_list(raw), r, s, recid


def get_senders(ctx, encoded_txs, chain_id=1):
    """TxSigner.get_sender (src/signer/signer.zig:41-79) for every transaction of a block: one K call for the signing
    hashes, one R call (phant_gpu_ecrecover_batch: recovery and address hashing fused) for the senders.  Returns a list
    with, per transaction, the 20-byte address or the SenderError the reference would have raised."""
    out = [None] * len(encoded_txs)
    parts = []
    for i, tx in enumerate(encoded_txs):
        try:
            parts.append((i,) + _tx_signing_parts(tx, chain_id))
        except SenderError as e:
            out[i] = e
    if not parts:
        return out
    hashes = keccak256_batch(ctx, [p[1] for p in parts])
    n = len(parts)
    h = np.frombuffer(b"".join(hashes), np.uint8)
    sig = np.frombuffer(b"".join(p[2].to_bytes(32, "big") + p[3].to_bytes(32, "big") + bytes([p[4]]) for p in parts), np.uint8)
    addr = np.zeros((n, 20), np.uint8)
    ok = np.zeros(n, np.uint8)
    ctx.ecrecover_batch(h, sig, n, None, addr, ok)
    for j, p in enumerate(parts):
        out[p[0]] = addr[j].tobytes() if ok[j] else SenderError("RecoveryFailed")
    return out


# ---- the payload handler with its TODO filled in (src/engine_api/execution_payload.zig:125-183) -------------------------------
def new_payload_v2(ctx, transactions, withdrawals, witness=None, parent_state_root=None, touched_hashed_keys=(), chain_id=1):
    """What newPayloadV2Handler does before it hands the block to runBlock, as three library calls for the whole payload:

      * ExecutionPayload.toBlock's two tries (:125-158; keys are the 32-byte big-endian index, phant's non-standard choice)
        built as ONE forest (M);
      * "reconstruct the proof from the execution witness and verify it" (:177-178): the witness blob decoded and every
        touched key resolved inside its node set from the parent state root (W);
      * the senders of all transactions (signer.zig:41-79) in one recovery call (R).

    transactions / withdrawals: encoded items.  Returns a dict; `accept` is False when the witness is undecodable or any
    touched key is rejected (0) or lacks a node (3) -- the payload must then be refused before execution."""
    if transactions or withdrawals:
        tx_root, wd_root = mptize_many(ctx, [[KeyVal(i.to_bytes(32, "big"), v) for i, v in enumerate(items)] for items in (transactions, withdrawals)])
    else:
        tx_root = wd_root = EMPTY_MPT_ROOT  # mpt.zig:41: an empty list hashes to the constant
    out = {"transactions_root": tx_root, "withdrawals_root": wd_root, "witness_status": None, "witness_error": None,
           "senders": get_senders(ctx, transactions, chain_id), "accept": True}
    if witness is not None:
        try:
            out["witness_status"] = verify_payload_witness(ctx, parent_state_root, witness, list(touched_hashed_keys))
            out["accept"] = all(s in (1, 2) for s in out["witness_status"])
        except InvalidWitness as e:
            out["witness_error"], out["accept"] = str(e), False
    return out


def transition_root(ctx, parent_root, witness_blob, touched, changed_slots=None, recreated=()):
    """The post-state root a stateless client checks against the block header: the witness blob decoded, the block's changes
    hashed exactly as ResidentStateDB.apply takes them, then ONE transition-roots call (phant_gpu_transition_roots) that
    applies them to the witness's paths under `parent_root` and rebuilds the tries on the device.  Returns (root, status):
    status 1 and the root, or status 0 (a node breaks the rules) / 3 (the witness lacks a node the computation needs) and
    None.  Raises InvalidWitness for an undecodable blob."""
    _, _, nodes = decode_witness(witness_blob)
    ndata, noff = _csr(list(nodes), np.uint64)
    pre = np.frombuffer(bytes(parent_root), np.uint8)
    if touched:
        d = _hashed_diff(ctx, touched, changed_slots, recreated)
    else:
        empty = np.zeros(0, np.uint8)
        d = dict(account_keys32=empty, nonce=np.zeros(0, np.uint64), balance32=empty, code_hash32=empty)
    roots, status = ctx.transition_roots(ndata, noff, pre, **d)
    return (roots[0].tobytes() if status[0] == 1 else None), int(status[0])


def _proof_csr(proof_nodes):
    """a ResidentState.prove batch (its `nodes` / `node_off`) or a list of node bytes -> the node set as CSR"""
    if isinstance(proof_nodes, dict):
        return np.ascontiguousarray(proof_nodes["nodes"], np.uint8), np.ascontiguousarray(proof_nodes["node_off"], np.uint64)
    return _csr(list(proof_nodes), np.uint64)


def verify_ranges(ctx, ranges, proof_nodes):
    """range proofs checked on the GPU, many in one call (phant_gpu_verify_ranges, DESIGN.md §4.3j).  ranges: [(root32,
    origin32, [(hashed key, leaf value bytes)], whole)], the entries ascending; proof_nodes: the boundary proofs of every
    range that is not whole, one node set.  Returns [(status, more)]: status 1 when the entries are exactly the trie's
    contents from the origin to the last entry (all of it when whole), 0 when they are not, 3 when a node is missing;
    more: the trie holds a key after the last entry."""
    nodes, noff = _proof_csr(proof_nodes)
    n = len(ranges)
    entries = [e for r in ranges for e in r[2]]
    first = np.zeros(n + 1, np.uint64)
    first[1:] = np.cumsum([len(r[2]) for r in ranges])
    keys = np.frombuffer(b"".join(k for k, _ in entries), np.uint8) if entries else np.zeros(32, np.uint8)
    vals, voff = _csr([v for _, v in entries], np.uint64)
    roots = np.frombuffer(b"".join(r[0] for r in ranges), np.uint8)
    origins = np.frombuffer(b"".join(r[1] for r in ranges), np.uint8)
    flags = np.array([gpu.RANGE_WHOLE if r[3] else 0 for r in ranges], np.uint8)
    status, more = ctx.verify_ranges(nodes, noff, roots, origins, first, keys[:32 * len(entries)], vals, voff, flags)
    return [(int(s), bool(m)) for s, m in zip(status, more)]


def _account_value(a):
    """an account_range entry's leaf value: rlp([nonce, balance, storageRoot, codeHash])"""
    return _rlp_list([_rlp_uint(a["nonce"]), _rlp_uint(a["balance"]), _rlp_str(a["storageHash"]), _rlp_str(a["codeHash"])])


def verify_account_range(ctx, root, origin, accounts, proof_nodes):
    """snap's check of a GetAccountRange answer against the state root: accounts as ResidentStateDB.account_range_proof
    returns them ([(hashed address, {nonce, balance, storageHash, codeHash})]) and its `proof`.  Returns (ok, more): ok when
    the accounts are exactly the state's accounts from `origin` to the last of them; more when accounts follow it."""
    (st, more), = verify_ranges(ctx, [(root, origin, [(k, _account_value(a)) for k, a in accounts], False)], proof_nodes)
    return st == 1, more


def verify_storage_ranges(ctx, ranges, proof_nodes, last_is_partial):
    """snap's check of a GetStorageRanges answer: ranges [(storage root, origin, slots)], slots as storage_range_proof
    returns them ([(hashed slot, value)]).  Every range but the last is a whole storage trie; the last is too unless
    last_is_partial, when proof_nodes (storage_range_proof's `proof`) prove it from its origin.  Returns [(ok, more)]."""
    rs = [(sroot, origin, [(k, _rlp_str(int(v).to_bytes(32, "big").lstrip(b"\x00"))) for k, v in slots],
           not (last_is_partial and i + 1 == len(ranges))) for i, (sroot, origin, slots) in enumerate(ranges)]
    return [(st == 1, more) for st, more in verify_ranges(ctx, rs, proof_nodes if last_is_partial else [])] if rs else []


def decode_slim_account(body):
    """a snap slim account body rlp([nonce, balance, storageRoot or "", codeHash or ""]) -> (nonce, balance, storageRoot,
    codeHash), the empty fields expanded to the empty root and keccak(""); raises InvalidWitness when it does not decode"""
    body = bytes(body)
    is_list, ps, pe = _rlp_header(body, 0, len(body))
    items = _rlp_list_items(body, ps, pe) if is_list and pe == len(body) else []
    if len(items) != 4 or any(it[0] for it in items):
        raise InvalidWitness("a slim account body is a list of four strings")
    f = [body[s:e] for _, _, s, e in items]
    if len(f[0]) > 8 or len(f[1]) > 32 or (f[0][:1] == b"\x00") or (f[1][:1] == b"\x00") or len(f[2]) not in (0, 32) or len(f[3]) not in (0, 32):
        raise InvalidWitness("a slim account field has the wrong length")
    return (int.from_bytes(f[0], "big"), int.from_bytes(f[1], "big"), f[2] or EMPTY_MPT_ROOT, f[3] or EMPTY_CODE_HASH)


def _full_account(body):
    nonce, balance, sroot, code = decode_slim_account(body)
    return _rlp_list([_rlp_uint(nonce), _rlp_uint(balance), _rlp_str(sroot), _rlp_str(code)])


def verify_snap_account_range(ctx, root, origin, accounts, proof):
    """a syncing peer's check of a GetAccountRange answer as it comes off the wire (snap_account_range's): the slim bodies
    expanded to the trie's leaves and checked with G from `origin`.  Returns (ok, more): more when accounts follow the last."""
    (st, more), = verify_ranges(ctx, [(root, origin, [(k, _full_account(b)) for k, b in accounts], False)], proof)
    return st == 1, more


def verify_snap_storage_ranges(ctx, storage_roots, origin, slots, proof):
    """a syncing peer's check of a GetStorageRanges answer (snap_storage_ranges's) with G: storage_roots of the served
    accounts, in order.  Every list is checked whole against its root, except the last when the answer carries a proof:
    that one is checked from its origin (the request's origin for the first account, else 0).  Returns [(ok, more)]."""
    rs = []
    for i, (sroot, lst) in enumerate(zip(storage_roots, slots)):
        partial = bool(proof) and i + 1 == len(slots)
        rs.append((bytes(sroot), bytes(origin) if i == 0 else bytes(32), [(bytes(k), bytes(v)) for k, v in lst], not partial))
    return [(st == 1, more) for st, more in verify_ranges(ctx, rs, proof)] if rs else []
