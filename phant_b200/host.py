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


class ResidentStateDB:
    """StateDB.root() block after block with the world state resident on the device (gpu.ResidentState, DESIGN.md §4.3c):
    addresses, slot numbers and code are hashed with K, the diff is built from the touched accounts and the changed slots,
    and one apply returns the new root.  No storage root is computed on the host."""

    def __init__(self, ctx):
        self.ctx = ctx
        self.state = ctx.resident_state()
        self.journal = 0

    def set_journal(self, depth):
        """keep what undoes each of the last `depth` applies on the device, so that revert() can take blocks back"""
        self.state.set_journal(depth)
        self.journal = depth

    def revert(self, n=1):
        """undo the last n applies (a block whose root did not match its header, or the blocks a reorg leaves); returns the
        root before the oldest of them"""
        return self.state.revert(n)

    def load(self, statedb):
        """the first apply: every account of `statedb` with all its slots"""
        return self.apply(statedb.db)

    def apply(self, touched, changed_slots=None, recreated=()):
        """touched: address -> AccountState, or None for a destroyed account.  changed_slots: address -> {slot: new value}
        (0 = deleted) for the slots the block wrote, every address in it touched and live; None = send each touched
        account's whole storage in place of what the device holds (CLEAR_STORAGE).  recreated: addresses (touched, live)
        destroyed and created again in the block: their old storage is dropped before their changed slots apply."""
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
        block's codes, encode_witness turns them into the blob transition_root reads."""
        if not touched:
            return []
        d = _hashed_diff(self.ctx, touched, changed_slots, recreated)
        nodes, off = self.state.witness(**d)
        return [nodes[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]

    def close(self):
        self.state.close()


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
