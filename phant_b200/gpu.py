"""ctypes binding of include/phant_gpu.h (libphantgpu.so).  Fails loudly when the library is missing."""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libphantgpu.so")

FLAG_DEVICE_PTRS = 1 << 0
FLAG_KECCAK_DIRECT = 1 << 4
FLAG_KECCAK_WARP = 1 << 5
FLAG_NO_BINNING = 1 << 6
FLAG_UNFUSED_WALK = 1 << 7

u8p, u32p, u64p = C.POINTER(C.c_uint8), C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)


class PhantGpuError(RuntimeError):
    def __init__(self, code, where, detail=""):
        self.code = code
        super().__init__(f"{where}: {_lib().phant_gpu_strerror(code).decode()} ({code}) {detail}")


class Config(C.Structure):
    _fields_ = [("device", C.c_int32), ("flags", C.c_uint32), ("reserved", C.c_uint64 * 4)]


class Stats(C.Structure):
    _fields_ = [("launches", C.c_uint64), ("h2d_bytes", C.c_uint64), ("d2h_bytes", C.c_uint64), ("keccak_ms", C.c_double),
                ("walk_ms", C.c_double), ("keccak_msgs", C.c_uint64), ("keccak_bytes", C.c_uint64), ("keccak_perms", C.c_uint64),
                ("reserved", C.c_uint64 * 4)]


class Accounts(C.Structure):
    _fields_ = [("n_accounts", C.c_uint64), ("addr20", C.c_void_p), ("nonce", C.c_void_p), ("balance32", C.c_void_p),
                ("code", C.c_void_p), ("code_off", C.c_void_p), ("slot_keys32", C.c_void_p), ("slot_vals32", C.c_void_p),
                ("slot_off", C.c_void_p)]


class ProofBatch(C.Structure):
    _fields_ = [("n_proofs", C.c_uint64), ("nodes", C.c_void_p), ("node_off", C.c_void_p), ("proof_first", C.c_void_p),
                ("keys32", C.c_void_p), ("roots32", C.c_void_p), ("n_roots", C.c_uint64), ("n_nodes", C.c_uint64),
                ("nodes_bytes", C.c_uint64), ("node_index", C.c_void_p)]


class Witness(C.Structure):
    _fields_ = [("n_nodes", C.c_uint64), ("nodes", C.c_void_p), ("node_off", C.c_void_p), ("nodes_bytes", C.c_uint64),
                ("n_keys", C.c_uint64), ("keys32", C.c_void_p), ("roots32", C.c_void_p), ("n_roots", C.c_uint64)]


class StateReads(C.Structure):
    _fields_ = [("n_nodes", C.c_uint64), ("nodes", C.c_void_p), ("node_off", C.c_void_p), ("nodes_bytes", C.c_uint64),
                ("n_codes", C.c_uint64), ("codes", C.c_void_p), ("code_off", C.c_void_p), ("codes_bytes", C.c_uint64),
                ("roots32", C.c_void_p), ("n_roots", C.c_uint64), ("n_accounts", C.c_uint64), ("account_keys32", C.c_void_p),
                ("n_slots", C.c_uint64), ("slot_keys32", C.c_void_p), ("slot_account", C.c_void_p)]


class StateValues(C.Structure):
    _fields_ = [("account_status", C.c_void_p), ("nonce", C.c_void_p), ("balance32", C.c_void_p), ("storage_root32", C.c_void_p),
                ("code_hash32", C.c_void_p), ("code_index", C.c_void_p), ("slot_status", C.c_void_p), ("slot_vals32", C.c_void_p)]


CODE_EMPTY = 0xFFFFFFFF    # PHANT_GPU_CODE_EMPTY: codeHash == keccak(""), or the account is not present
CODE_MISSING = 0xFFFFFFFE  # PHANT_GPU_CODE_MISSING: no witness code hashes to the account's codeHash


class TrieDesc(C.Structure):
    _fields_ = [("kind", C.c_uint32), ("depth", C.c_uint32), ("seed", C.c_uint64), ("reserved", C.c_uint64 * 4)]


class StateDiff(C.Structure):
    _fields_ = [("n_accounts", C.c_uint64), ("account_keys32", C.c_void_p), ("account_flags", C.c_void_p), ("nonce", C.c_void_p),
                ("balance32", C.c_void_p), ("code_hash32", C.c_void_p), ("n_slots", C.c_uint64), ("slot_account", C.c_void_p),
                ("slot_keys32", C.c_void_p), ("slot_vals32", C.c_void_p)]


class StateInfo(C.Structure):
    _fields_ = [("n_accounts", C.c_uint64), ("n_slots", C.c_uint64), ("device_bytes", C.c_uint64), ("journal_applies", C.c_uint64),
                ("journal_bytes", C.c_uint64), ("reserved", C.c_uint64 * 2)]


class WitnessSize(C.Structure):
    _fields_ = [("n_nodes", C.c_uint64), ("nodes_bytes", C.c_uint64), ("reserved", C.c_uint64 * 2)]


class Transition(C.Structure):
    _fields_ = [("n_nodes", C.c_uint64), ("nodes", C.c_void_p), ("node_off", C.c_void_p), ("nodes_bytes", C.c_uint64),
                ("n_blocks", C.c_uint64), ("pre_roots32", C.c_void_p), ("account_block", C.c_void_p)]


ACCOUNT_DELETE = 1         # PHANT_GPU_ACCOUNT_DELETE: remove the account and all of its storage
ACCOUNT_CLEAR_STORAGE = 2  # PHANT_GPU_ACCOUNT_CLEAR_STORAGE: drop its storage before the diff's slots (re-created account)


EXPORTS = [
    "phant_gpu_abi_version", "phant_gpu_create", "phant_gpu_destroy", "phant_gpu_set_flags", "phant_gpu_set_stream", "phant_gpu_strerror",
    "phant_gpu_last_error", "phant_gpu_get_stats", "phant_gpu_reset_stats", "phant_gpu_synchronize",
    "phant_gpu_keccak256_batch", "phant_gpu_keccak256_batch_async", "phant_gpu_mpt_root", "phant_gpu_mpt_roots", "phant_gpu_state_root", "phant_gpu_state_subtree_roots", "phant_gpu_ecrecover_batch", "phant_gpu_verify_proofs", "phant_gpu_verify_witness",
    "phant_gpu_read_state",
    "phant_gpu_logs_bloom", "phant_gpu_trie_open", "phant_gpu_trie_root", "phant_gpu_trie_update", "phant_gpu_trie_close",
    "phant_gpu_resident_state_open", "phant_gpu_resident_state_apply", "phant_gpu_resident_state_root", "phant_gpu_resident_state_info",
    "phant_gpu_resident_state_close", "phant_gpu_resident_state_set_journal", "phant_gpu_resident_state_revert",
    "phant_gpu_resident_state_witness", "phant_gpu_resident_state_witness_copy", "phant_gpu_transition_roots",
    "phant_gpu_synth_sizes", "phant_gpu_synth",
    "phant_gpu_comm_get_unique_id", "phant_gpu_comm_init", "phant_gpu_comm_init_local", "phant_gpu_comm_info", "phant_gpu_comm_enable_peer", "phant_gpu_comm_disable_peer", "phant_gpu_comm_peer_status", "phant_gpu_comm_fence",
    "phant_gpu_comm_destroy", "phant_gpu_shard_range", "phant_gpu_sharded_bitmap_words", "phant_gpu_verify_proofs_sharded",
    "phant_gpu_block_reject_counts", "phant_gpu_nibble_owner", "phant_gpu_state_root_sharded",
]
COMM_ID_BYTES = 128

_LIB = None


def _lib():
    global _LIB
    if _LIB is not None:
        return _LIB
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(there is no CPU fallback)")
    L = C.CDLL(LIB_PATH)
    vp = C.c_void_p
    L.phant_gpu_abi_version.restype = C.c_int
    L.phant_gpu_create.argtypes = [C.POINTER(vp), C.POINTER(Config)]
    L.phant_gpu_destroy.argtypes = [vp]
    L.phant_gpu_destroy.restype = None
    L.phant_gpu_set_flags.argtypes = [vp, C.c_uint32]
    L.phant_gpu_set_stream.argtypes = [vp, vp]
    L.phant_gpu_strerror.argtypes = [C.c_int]
    L.phant_gpu_strerror.restype = C.c_char_p
    L.phant_gpu_last_error.argtypes = [vp]
    L.phant_gpu_last_error.restype = C.c_char_p
    L.phant_gpu_get_stats.argtypes = [vp, C.POINTER(Stats)]
    L.phant_gpu_reset_stats.argtypes = [vp]
    L.phant_gpu_synchronize.argtypes = [vp]
    L.phant_gpu_keccak256_batch.argtypes = [vp, vp, vp, C.c_uint64, vp]
    L.phant_gpu_keccak256_batch_async.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint64, vp]
    L.phant_gpu_mpt_root.argtypes = [vp, vp, vp, vp, vp, C.c_uint64, vp]
    L.phant_gpu_mpt_roots.argtypes = [vp, vp, vp, vp, vp, vp, C.c_uint64, vp]
    L.phant_gpu_state_root.argtypes = [vp, C.POINTER(Accounts), vp]
    L.phant_gpu_state_subtree_roots.argtypes = [vp, C.POINTER(Accounts), vp, C.POINTER(C.c_uint32)]
    L.phant_gpu_ecrecover_batch.argtypes = [vp, vp, vp, C.c_uint64, vp, vp, vp]
    L.phant_gpu_verify_proofs.argtypes = [vp, C.POINTER(ProofBatch), vp, vp, vp, vp]
    L.phant_gpu_verify_witness.argtypes = [vp, C.POINTER(Witness), vp, vp, vp, vp]
    L.phant_gpu_read_state.argtypes = [vp, C.POINTER(StateReads), C.POINTER(StateValues)]
    L.phant_gpu_logs_bloom.argtypes = [vp, vp, vp, vp, C.c_uint64, C.c_uint64, vp]
    L.phant_gpu_trie_open.argtypes = [vp, C.POINTER(TrieDesc), C.POINTER(vp)]
    L.phant_gpu_trie_root.argtypes = [vp, vp]
    L.phant_gpu_trie_update.argtypes = [vp, vp, vp, vp, C.c_uint64, vp]
    L.phant_gpu_trie_close.argtypes = [vp]
    L.phant_gpu_trie_close.restype = None
    L.phant_gpu_resident_state_open.argtypes = [vp, C.POINTER(vp)]
    L.phant_gpu_resident_state_apply.argtypes = [vp, C.POINTER(StateDiff), vp, vp]
    L.phant_gpu_resident_state_root.argtypes = [vp, vp]
    L.phant_gpu_resident_state_info.argtypes = [vp, C.POINTER(StateInfo)]
    L.phant_gpu_resident_state_close.argtypes = [vp]
    L.phant_gpu_resident_state_close.restype = None
    L.phant_gpu_resident_state_set_journal.argtypes = [vp, C.c_uint32]
    L.phant_gpu_resident_state_revert.argtypes = [vp, C.c_uint32, vp]
    L.phant_gpu_resident_state_witness.argtypes = [vp, C.POINTER(StateDiff), C.POINTER(WitnessSize)]
    L.phant_gpu_resident_state_witness_copy.argtypes = [vp, vp, vp]
    L.phant_gpu_transition_roots.argtypes = [vp, C.POINTER(Transition), C.POINTER(StateDiff), vp, vp, vp]
    L.phant_gpu_synth_sizes.argtypes = [vp, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, u64p, u64p]
    L.phant_gpu_synth.argtypes = [vp, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_int, vp, vp, vp, vp, vp]
    L.phant_gpu_comm_get_unique_id.argtypes = [vp]
    L.phant_gpu_comm_init.argtypes = [vp, vp, C.c_int, C.c_int]
    L.phant_gpu_comm_init_local.argtypes = [C.POINTER(vp), C.c_int]
    L.phant_gpu_comm_info.argtypes = [vp, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.phant_gpu_comm_enable_peer.argtypes = [vp, C.c_uint64]
    L.phant_gpu_comm_disable_peer.argtypes = [vp]
    L.phant_gpu_comm_peer_status.argtypes = [vp, C.POINTER(C.c_int), u64p, C.POINTER(C.c_int)]
    L.phant_gpu_comm_fence.argtypes = [vp]
    L.phant_gpu_comm_destroy.argtypes = [vp]
    L.phant_gpu_shard_range.argtypes = [C.c_uint64, C.c_int, C.c_int, u64p, u64p]
    L.phant_gpu_sharded_bitmap_words.argtypes = [C.c_uint64, C.c_int]
    L.phant_gpu_sharded_bitmap_words.restype = C.c_uint64
    L.phant_gpu_verify_proofs_sharded.argtypes = [vp, C.POINTER(ProofBatch), C.c_uint64, vp, vp, vp, vp]
    L.phant_gpu_block_reject_counts.argtypes = [vp, vp, vp, C.c_uint64, C.c_uint64, vp]
    L.phant_gpu_nibble_owner.argtypes = [C.c_int, C.c_int]
    L.phant_gpu_state_root_sharded.argtypes = [vp, C.POINTER(Accounts), vp]
    _LIB = L
    return L


def _ptr(a):
    """numpy array / torch tensor / int / None -> raw address"""
    if a is None:
        return None
    if isinstance(a, int):
        return a
    if isinstance(a, np.ndarray):
        assert a.flags["C_CONTIGUOUS"]
        return a.ctypes.data
    return a.data_ptr()  # torch tensor


class Context:
    """One device, one stream (phant_gpu_ctx).  Not thread safe."""

    def __init__(self, device=0, flags=0):
        self._h = C.c_void_p()
        cfg = Config(device, flags)
        rc = _lib().phant_gpu_create(C.byref(self._h), C.byref(cfg))
        if rc != 0:
            self._h = None
            raise PhantGpuError(rc, "phant_gpu_create")
        self.device = device
        self.flags = flags

    def close(self):
        for t in list(getattr(self, "_tries", [])):
            t.close()
        if getattr(self, "_h", None):
            _lib().phant_gpu_destroy(self._h)
            self._h = None

    __del__ = close

    def _chk(self, rc, where):
        if rc != 0:
            raise PhantGpuError(rc, where, _lib().phant_gpu_last_error(self._h).decode())

    def set_flags(self, flags):
        self._chk(_lib().phant_gpu_set_flags(self._h, flags), "set_flags")
        self.flags = flags

    def set_stream(self, cuda_stream):
        """cuda_stream: integer handle (e.g. torch.cuda.current_stream().cuda_stream) or None"""
        self._chk(_lib().phant_gpu_set_stream(self._h, cuda_stream), "set_stream")

    def synchronize(self):
        self._chk(_lib().phant_gpu_synchronize(self._h), "synchronize")

    def stats(self):
        s = Stats()
        self._chk(_lib().phant_gpu_get_stats(self._h, C.byref(s)), "get_stats")
        return {k: getattr(s, k) for k, _ in Stats._fields_ if k != "reserved"}

    def reset_stats(self):
        self._chk(_lib().phant_gpu_reset_stats(self._h), "reset_stats")

    # K
    def keccak256_batch(self, msgs, off, n, out):
        self._chk(_lib().phant_gpu_keccak256_batch(self._h, _ptr(msgs), _ptr(off), n, _ptr(out)), "keccak256_batch")

    def keccak256_batch_async(self, msgs, off, n, total_bytes, out):
        """device pointers, total supplied: no read-back, asynchronous on the context's stream"""
        self._chk(_lib().phant_gpu_keccak256_batch_async(self._h, _ptr(msgs), _ptr(off), n, total_bytes, _ptr(out)), "keccak256_batch_async")

    # M
    def mpt_root(self, keys, key_off, vals, val_off, n):
        out = np.zeros(32, np.uint8)
        self._chk(_lib().phant_gpu_mpt_root(self._h, _ptr(keys), _ptr(key_off), _ptr(vals), _ptr(val_off), n, _ptr(out)), "mpt_root")
        return out.tobytes()

    def mpt_roots(self, keys, key_off, vals, val_off, seg_off, n_tries):
        out = np.zeros((max(n_tries, 1), 32), np.uint8)
        self._chk(_lib().phant_gpu_mpt_roots(self._h, _ptr(keys), _ptr(key_off), _ptr(vals), _ptr(val_off), _ptr(seg_off), n_tries, _ptr(out)),
                  "mpt_roots")
        return [out[i].tobytes() for i in range(n_tries)]

    # S
    def state_root(self, n, addr20, nonce, balance32, code, code_off, slot_keys32, slot_vals32, slot_off):
        a = Accounts(n, _ptr(addr20), _ptr(nonce), _ptr(balance32), _ptr(code), _ptr(code_off), _ptr(slot_keys32),
                     _ptr(slot_vals32), _ptr(slot_off))
        out = np.zeros(32, np.uint8)
        self._chk(_lib().phant_gpu_state_root(self._h, C.byref(a), _ptr(out)), "state_root")
        return out.tobytes()

    def state_subtree_roots(self, n, addr20, nonce, balance32, code, code_off, slot_keys32, slot_vals32, slot_off):
        """(16 x 32 uint8 subtree hashes under the root branch, populated-slot mask) of the accounts handed in"""
        a = Accounts(n, _ptr(addr20), _ptr(nonce), _ptr(balance32), _ptr(code), _ptr(code_off), _ptr(slot_keys32),
                     _ptr(slot_vals32), _ptr(slot_off))
        out = np.zeros((16, 32), np.uint8)
        mask = C.c_uint32(0)
        self._chk(_lib().phant_gpu_state_subtree_roots(self._h, C.byref(a), _ptr(out), C.byref(mask)), "state_subtree_roots")
        return out, int(mask.value)

    # R
    def ecrecover_batch(self, hashes32, sigs65, n, pubkeys65=None, addresses20=None, ok=None):
        self._chk(_lib().phant_gpu_ecrecover_batch(self._h, _ptr(hashes32), _ptr(sigs65), n, _ptr(pubkeys65), _ptr(addresses20), _ptr(ok)),
                  "ecrecover_batch")

    # V
    def verify_proofs(self, n_proofs, nodes, node_off, proof_first, keys32, roots32, n_roots, bitmap=None, status=None,
                      val_off=None, val_len=None, n_nodes=0, nodes_bytes=0, node_index=None):
        b = ProofBatch(n_proofs, _ptr(nodes), _ptr(node_off), _ptr(proof_first), _ptr(keys32), _ptr(roots32), n_roots,
                       n_nodes, nodes_bytes, _ptr(node_index))
        self._chk(_lib().phant_gpu_verify_proofs(self._h, C.byref(b), _ptr(bitmap), _ptr(status), _ptr(val_off), _ptr(val_len)),
                  "verify_proofs")

    # W
    def verify_witness(self, n_nodes, nodes, node_off, n_keys, keys32, roots32, n_roots, bitmap=None, status=None, val_off=None,
                       val_len=None, nodes_bytes=0):
        w = Witness(n_nodes, _ptr(nodes), _ptr(node_off), nodes_bytes, n_keys, _ptr(keys32), _ptr(roots32), n_roots)
        self._chk(_lib().phant_gpu_verify_witness(self._h, C.byref(w), _ptr(bitmap), _ptr(status), _ptr(val_off), _ptr(val_len)),
                  "verify_witness")

    # P
    def read_state(self, n_nodes, nodes, node_off, n_accounts, account_keys32, roots32, n_roots, n_slots=0, slot_keys32=None,
                   slot_account=None, n_codes=0, codes=None, code_off=None, nodes_bytes=0, codes_bytes=0, account_status=None, nonce=None,
                   balance32=None, storage_root32=None, code_hash32=None, code_index=None, slot_status=None, slot_vals32=None):
        """pre-state reads (phant_gpu_read_state): every output may be None"""
        r = StateReads(n_nodes, _ptr(nodes), _ptr(node_off), nodes_bytes, n_codes, _ptr(codes), _ptr(code_off), codes_bytes, _ptr(roots32),
                       n_roots, n_accounts, _ptr(account_keys32), n_slots, _ptr(slot_keys32), _ptr(slot_account))
        v = StateValues(_ptr(account_status), _ptr(nonce), _ptr(balance32), _ptr(storage_root32), _ptr(code_hash32), _ptr(code_index),
                        _ptr(slot_status), _ptr(slot_vals32))
        self._chk(_lib().phant_gpu_read_state(self._h, C.byref(r), C.byref(v)), "read_state")

    # B
    # T
    def transition_roots(self, nodes, node_off, pre_roots32, account_keys32, nonce, balance32, code_hash32, account_flags=None,
                         account_block=None, slot_account=None, slot_keys32=None, slot_vals32=None, storage_roots=False):
        """post-state root of each block from a witness node set (CSR) and a diff (phant_gpu_transition_roots).  pre_roots32:
        n_blocks x 32; account_block: the block of each listed account (None: all in block 0).  Returns (roots n_blocks x 32,
        status n_blocks), plus the listed accounts' storage roots (n x 32) when storage_roots is true."""
        pre = np.ascontiguousarray(pre_roots32, dtype=np.uint8).reshape(-1, 32)
        nb = pre.shape[0]
        n = len(nonce)
        ak = _u8_rows(account_keys32, n, 32)
        nn = np.ascontiguousarray(nonce, dtype=np.uint64)
        bal = _u8_rows(balance32, n, 32)
        ch = _u8_rows(code_hash32, n, 32)
        fl = None if account_flags is None else np.ascontiguousarray(account_flags, dtype=np.uint8)
        ab = None if account_block is None else np.ascontiguousarray(account_block, dtype=np.uint32)
        m = 0 if slot_account is None else len(slot_account)
        sa = None if not m else np.ascontiguousarray(slot_account, dtype=np.uint32)
        sk = None if not m else _u8_rows(slot_keys32, m, 32)
        sv = None if not m else _u8_rows(slot_vals32, m, 32)
        off = np.ascontiguousarray(node_off, dtype=np.uint64)
        data = np.ascontiguousarray(nodes, dtype=np.uint8)
        t = Transition(len(off) - 1, _ptr(data), _ptr(off), int(off[-1]), nb, _ptr(pre), _ptr(ab))
        d = StateDiff(n, _ptr(ak), _ptr(fl), _ptr(nn), _ptr(bal), _ptr(ch), m, _ptr(sa), _ptr(sk), _ptr(sv))
        roots = np.zeros((nb, 32), np.uint8)
        status = np.zeros(nb, np.uint8)
        sroots = np.zeros((max(n, 1), 32), np.uint8) if storage_roots else None
        self._chk(_lib().phant_gpu_transition_roots(self._h, C.byref(t), C.byref(d), _ptr(roots), _ptr(status), _ptr(sroots)),
                  "transition_roots")
        return (roots, status, sroots[:n]) if storage_roots else (roots, status)

    def transition_roots_raw(self, t, d, roots, status, sroots=None):
        """structs and buffers built by the caller: the return code, not an exception"""
        return _lib().phant_gpu_transition_roots(self._h, C.byref(t), C.byref(d), _ptr(roots), _ptr(status), _ptr(sroots))

    def logs_bloom(self, items, item_off, bloom_of_item, n_items, n_blooms, blooms):
        self._chk(_lib().phant_gpu_logs_bloom(self._h, _ptr(items), _ptr(item_off), _ptr(bloom_of_item), n_items, n_blooms, _ptr(blooms)),
                  "logs_bloom")

    # U
    def trie_open(self, depth, seed=0x5048414E54, kind=0):
        return ResidentTrie(self, depth, seed, kind)

    def resident_state(self):
        return ResidentState(self)

    # multi-GPU (comm.cu)
    def comm_init(self, unique_id, rank, world):
        """collective: every rank passes the id rank 0 got from comm_unique_id()"""
        buf = np.frombuffer(bytes(unique_id), np.uint8).copy()
        self._chk(_lib().phant_gpu_comm_init(self._h, _ptr(buf), rank, world), "comm_init")

    def comm_info(self):
        r, w, v = C.c_int(), C.c_int(), C.c_int()
        self._chk(_lib().phant_gpu_comm_info(self._h, C.byref(r), C.byref(w), C.byref(v)), "comm_info")
        return r.value, w.value, v.value

    def comm_enable_peer(self, max_n_global):
        """collective; afterwards equal-shard device-pointer calls of verify_proofs_sharded gather through peer memory
        (the walk's epilogue) instead of a NCCL launch.  Raises PhantGpuError(-5) when a mapping is impossible: NCCL stays."""
        self._chk(_lib().phant_gpu_comm_enable_peer(self._h, max_n_global), "comm_enable_peer")

    def comm_disable_peer(self):
        """collective: unmap the peer regions, back to the NCCL gather"""
        self._chk(_lib().phant_gpu_comm_disable_peer(self._h), "comm_disable_peer")

    def comm_peer_status(self):
        e, st, to = C.c_int(), C.c_uint64(), C.c_int()
        self._chk(_lib().phant_gpu_comm_peer_status(self._h, C.byref(e), C.byref(st), C.byref(to)), "comm_peer_status")
        return {"enabled": bool(e.value), "steps": int(st.value), "timed_out": bool(to.value)}

    def comm_fence(self):
        self._chk(_lib().phant_gpu_comm_fence(self._h), "comm_fence")

    def comm_destroy(self):
        self._chk(_lib().phant_gpu_comm_destroy(self._h), "comm_destroy")

    def verify_proofs_sharded(self, n_local, n_global, nodes, node_off, proof_first, keys32, roots32, n_roots, global_bitmap, status=None,
                              val_off=None, val_len=None, n_nodes=0, nodes_bytes=0, node_index=None):
        b = ProofBatch(n_local, _ptr(nodes), _ptr(node_off), _ptr(proof_first), _ptr(keys32), _ptr(roots32), n_roots,
                       n_nodes, nodes_bytes, _ptr(node_index))
        self._chk(_lib().phant_gpu_verify_proofs_sharded(self._h, C.byref(b), n_global, _ptr(global_bitmap), _ptr(status), _ptr(val_off),
                                                         _ptr(val_len)), "verify_proofs_sharded")

    def block_reject_counts(self, status, block_of_proof, n_proofs, n_blocks, counts):
        self._chk(_lib().phant_gpu_block_reject_counts(self._h, _ptr(status), _ptr(block_of_proof), n_proofs, n_blocks, _ptr(counts)),
                  "block_reject_counts")

    def state_root_sharded(self, n, addr20, nonce, balance32, code, code_off, slot_keys32, slot_vals32, slot_off):
        a = Accounts(n, _ptr(addr20), _ptr(nonce), _ptr(balance32), _ptr(code), _ptr(code_off), _ptr(slot_keys32),
                     _ptr(slot_vals32), _ptr(slot_off))
        out = np.zeros(32, np.uint8)
        self._chk(_lib().phant_gpu_state_root_sharded(self._h, C.byref(a), _ptr(out)), "state_root_sharded")
        return out.tobytes()

    # synthetic (device pointers)
    def synth_sizes(self, which, n, depth=8, first=0, seed=0x5048414E54):
        a, b = C.c_uint64(), C.c_uint64()
        self._chk(_lib().phant_gpu_synth_sizes(self._h, which, seed, first, n, depth, C.byref(a), C.byref(b)), "synth_sizes")
        return a.value, b.value

    def synth(self, which, n, nodes, node_off, proof_first, keys32, roots32, depth=8, first=0, corrupt=True, seed=0x5048414E54):
        self._chk(_lib().phant_gpu_synth(self._h, which, seed, first, n, depth, int(corrupt), _ptr(nodes), _ptr(node_off),
                                         _ptr(proof_first), _ptr(keys32), _ptr(roots32)), "synth")


class ResidentTrie:
    def __init__(self, ctx, depth, seed, kind):
        self.ctx = ctx
        self._h = C.c_void_p()
        d = TrieDesc(kind, depth, seed)
        ctx._chk(_lib().phant_gpu_trie_open(ctx._h, C.byref(d), C.byref(self._h)), "trie_open")
        if not hasattr(ctx, "_tries"):
            ctx._tries = []
        ctx._tries.append(self)

    def root(self):
        out = np.zeros(32, np.uint8)
        self.ctx._chk(_lib().phant_gpu_trie_root(self._h, _ptr(out)), "trie_root")
        return out.tobytes()

    def update(self, keys32, leaf_vals, val_off, n_dirty):
        out = np.zeros(32, np.uint8)
        self.ctx._chk(_lib().phant_gpu_trie_update(self._h, _ptr(keys32), _ptr(leaf_vals), _ptr(val_off), n_dirty, _ptr(out)),
                      "trie_update")
        return out.tobytes()

    def close(self):
        if getattr(self, "_h", None) and getattr(self.ctx, "_h", None):
            _lib().phant_gpu_trie_close(self._h)
        self._h = None
        if self in getattr(self.ctx, "_tries", []):
            self.ctx._tries.remove(self)

    __del__ = close


def comm_unique_id():
    buf = np.zeros(COMM_ID_BYTES, np.uint8)
    rc = _lib().phant_gpu_comm_get_unique_id(_ptr(buf))
    if rc != 0:
        raise PhantGpuError(rc, "comm_get_unique_id", "(libnccl.so.2 not loadable? PHANT_GPU_NCCL_LIB overrides the name)")
    return buf.tobytes()


def comm_init_local(contexts):
    """one process, one context per device: rank i = contexts[i]; drive each from its own thread afterwards"""
    arr = (C.c_void_p * len(contexts))(*[c._h for c in contexts])
    rc = _lib().phant_gpu_comm_init_local(arr, len(contexts))
    if rc != 0:
        raise PhantGpuError(rc, "comm_init_local", _lib().phant_gpu_last_error(contexts[0]._h).decode())


def shard_range(n, rank, world):
    lo, hi = C.c_uint64(), C.c_uint64()
    rc = _lib().phant_gpu_shard_range(n, rank, world, C.byref(lo), C.byref(hi))
    if rc != 0:
        raise PhantGpuError(rc, "shard_range")
    return lo.value, hi.value


def sharded_bitmap_words(n, world):
    return int(_lib().phant_gpu_sharded_bitmap_words(n, world))


def nibble_owner(nibble, world):
    return int(_lib().phant_gpu_nibble_owner(nibble, world))


def abi_version():
    return _lib().phant_gpu_abi_version()


def exported_symbols():
    """every symbol include/phant_gpu.h declares that the loaded library really exports"""
    L = _lib()
    return [s for s in EXPORTS if hasattr(L, s)]


def _u8_rows(a, n, width):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.uint8)).reshape(-1)
    assert a.size == n * width, (a.size, n, width)
    return a


class ResidentState:
    """phant_gpu_resident_state: the account trie and every storage trie resident on the device (DESIGN.md §4.3c).
    apply() takes one block's changes with hashed keys; see StateDB-level helper phant_b200.host.ResidentStateDB."""

    def __init__(self, ctx):
        self.ctx = ctx
        self._h = C.c_void_p()
        ctx._chk(_lib().phant_gpu_resident_state_open(ctx._h, C.byref(self._h)), "resident_state_open")
        if not hasattr(ctx, "_tries"):
            ctx._tries = []
        ctx._tries.append(self)

    @staticmethod
    def _diff(account_keys32, nonce, balance32, code_hash32, account_flags, slot_account, slot_keys32, slot_vals32):
        n = len(nonce)
        ak = _u8_rows(account_keys32, n, 32)
        nn = np.ascontiguousarray(nonce, dtype=np.uint64)
        bal = _u8_rows(balance32, n, 32)
        ch = _u8_rows(code_hash32, n, 32)
        fl = None if account_flags is None else np.ascontiguousarray(account_flags, dtype=np.uint8)
        m = 0 if slot_account is None else len(slot_account)
        sa = None if not m else np.ascontiguousarray(slot_account, dtype=np.uint32)
        sk = None if not m else _u8_rows(slot_keys32, m, 32)
        sv = None if not m else _u8_rows(slot_vals32, m, 32)
        d = StateDiff(n, _ptr(ak), _ptr(fl), _ptr(nn), _ptr(bal), _ptr(ch), m, _ptr(sa), _ptr(sk), _ptr(sv))
        d._keep = (ak, nn, bal, ch, fl, sa, sk, sv)
        return d

    def apply(self, account_keys32, nonce, balance32, code_hash32, account_flags=None, slot_account=None, slot_keys32=None,
              slot_vals32=None, storage_roots=False):
        """numpy inputs: n x 32 uint8 keys / balances / code hashes, n uint64 nonces, n uint8 flags (or None); slots: uint32
        account indices, n_slots x 32 keys and values.  Returns the state root, or (root, n x 32 storage roots)."""
        d = self._diff(account_keys32, nonce, balance32, code_hash32, account_flags, slot_account, slot_keys32, slot_vals32)
        n = d.n_accounts
        out = np.zeros(32, np.uint8)
        roots = np.zeros((max(n, 1), 32), np.uint8) if storage_roots else None
        self.ctx._chk(_lib().phant_gpu_resident_state_apply(self._h, C.byref(d), _ptr(out), _ptr(roots)), "resident_state_apply")
        return (out.tobytes(), roots[:n]) if storage_roots else out.tobytes()

    def witness(self, account_keys32, nonce, balance32, code_hash32, account_flags=None, slot_account=None, slot_keys32=None,
                slot_vals32=None):
        """the pre-state execution witness of the diff apply() would take, from the state as it is now (which is not changed):
        (nodes, node_off), the node set as CSR, each node once, ordered by digest"""
        d = self._diff(account_keys32, nonce, balance32, code_hash32, account_flags, slot_account, slot_keys32, slot_vals32)
        size = WitnessSize()
        self.ctx._chk(_lib().phant_gpu_resident_state_witness(self._h, C.byref(d), C.byref(size)), "resident_state_witness")
        nodes = np.zeros(max(size.nodes_bytes, 1), np.uint8)
        off = np.zeros(size.n_nodes + 1, np.uint64)
        self.ctx._chk(_lib().phant_gpu_resident_state_witness_copy(self._h, _ptr(nodes), _ptr(off)), "resident_state_witness_copy")
        return nodes[:size.nodes_bytes], off

    def witness_raw(self, diff):
        """a StateDiff built by the caller: (return code, phant_gpu_witness_size)"""
        size = WitnessSize()
        return _lib().phant_gpu_resident_state_witness(self._h, C.byref(diff), C.byref(size)), size

    def witness_copy_raw(self, nodes, node_off):
        return _lib().phant_gpu_resident_state_witness_copy(self._h, _ptr(nodes), _ptr(node_off))

    def apply_raw(self, diff):
        """a StateDiff built by the caller (any pointers): the return code, not an exception"""
        out = np.zeros(32, np.uint8)
        return _lib().phant_gpu_resident_state_apply(self._h, C.byref(diff), _ptr(out), None)

    def root(self):
        out = np.zeros(32, np.uint8)
        self.ctx._chk(_lib().phant_gpu_resident_state_root(self._h, _ptr(out)), "resident_state_root")
        return out.tobytes()

    def info(self):
        i = StateInfo()
        self.ctx._chk(_lib().phant_gpu_resident_state_info(self._h, C.byref(i)), "resident_state_info")
        return {"n_accounts": i.n_accounts, "n_slots": i.n_slots, "device_bytes": i.device_bytes, "journal_applies": i.journal_applies,
                "journal_bytes": i.journal_bytes}

    def set_journal(self, depth):
        """keep the undo records of the last `depth` successful applies on the device (0: none)"""
        self.ctx._chk(_lib().phant_gpu_resident_state_set_journal(self._h, depth), "resident_state_set_journal")

    def revert(self, n=1):
        """undo the last n successful applies, newest first; returns the root before the oldest of them"""
        out = np.zeros(32, np.uint8)
        self.ctx._chk(_lib().phant_gpu_resident_state_revert(self._h, n, _ptr(out)), "resident_state_revert")
        return out.tobytes()

    def close(self):
        if getattr(self, "_h", None):
            _lib().phant_gpu_resident_state_close(self._h)
            self._h = None
        if self in getattr(self.ctx, "_tries", []):
            self.ctx._tries.remove(self)
