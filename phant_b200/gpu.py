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
                ("journal_bytes", C.c_uint64), ("n_codes", C.c_uint64), ("code_bytes", C.c_uint64)]


class WitnessSize(C.Structure):
    _fields_ = [("n_nodes", C.c_uint64), ("nodes_bytes", C.c_uint64), ("reserved", C.c_uint64 * 2)]


class ProofRequest(C.Structure):
    _fields_ = [("n_accounts", C.c_uint64), ("account_keys32", C.c_void_p), ("n_slots", C.c_uint64), ("slot_account", C.c_void_p),
                ("slot_keys32", C.c_void_p)]


class ProofSize(C.Structure):
    _fields_ = [("n_nodes", C.c_uint64), ("nodes_bytes", C.c_uint64), ("n_refs", C.c_uint64), ("reserved", C.c_uint64 * 2)]


class Proofs(C.Structure):
    _fields_ = [("nodes", C.c_void_p), ("node_off", C.c_void_p), ("node_index", C.c_void_p), ("proof_first", C.c_void_p),
                ("roots32", C.c_void_p), ("status", C.c_void_p), ("nonce", C.c_void_p), ("balance32", C.c_void_p),
                ("storage_root32", C.c_void_p), ("code_hash32", C.c_void_p), ("slot_vals32", C.c_void_p)]


class TrieNodeRequest(C.Structure):
    _fields_ = [("n_paths", C.c_uint64), ("paths32", C.c_void_p), ("path_len", C.c_void_p), ("path_trie", C.c_void_p),
                ("n_storage_accounts", C.c_uint64), ("storage_account32", C.c_void_p)]


class TrieNodes(C.Structure):
    _fields_ = [("status", C.c_void_p), ("node_off", C.c_void_p), ("nodes", C.c_void_p)]


class SnapRequest(C.Structure):
    _fields_ = [("n_account_requests", C.c_uint64), ("account_origin32", C.c_void_p), ("account_limit32", C.c_void_p),
                ("account_bytes", C.c_void_p), ("n_storage_requests", C.c_uint64), ("storage_first", C.c_void_p),
                ("storage_accounts32", C.c_void_p), ("storage_origin32", C.c_void_p), ("storage_limit32", C.c_void_p),
                ("storage_bytes", C.c_void_p)]


class SnapSize(C.Structure):
    _fields_ = [(f, C.c_uint64) for f in ("n_accounts", "account_bytes", "n_served", "n_slots", "slot_bytes", "n_nodes", "nodes_bytes",
                                          "n_refs")] + [("reserved", C.c_uint64 * 2)]


class SnapRanges(C.Structure):
    _fields_ = [(f, C.c_void_p) for f in ("account_first", "account_keys32", "account_body_off", "account_bodies", "served_first",
                                          "slot_first", "slot_keys32", "slot_body_off", "slot_bodies", "proof_first", "node_index",
                                          "nodes", "node_off")]


class StateReadValues(C.Structure):
    _fields_ = [("account_status", C.c_void_p), ("nonce", C.c_void_p), ("balance32", C.c_void_p), ("storage_root32", C.c_void_p),
                ("code_hash32", C.c_void_p), ("slot_status", C.c_void_p), ("slot_vals32", C.c_void_p)]


class RangeRequest(C.Structure):
    _fields_ = [("n_account_ranges", C.c_uint64), ("account_origin32", C.c_void_p), ("account_limit32", C.c_void_p),
                ("account_max", C.c_void_p), ("n_storage_ranges", C.c_uint64), ("storage_account32", C.c_void_p),
                ("storage_origin32", C.c_void_p), ("storage_limit32", C.c_void_p), ("storage_max", C.c_void_p)]


class RangeValues(C.Structure):
    _fields_ = [(f, C.c_void_p) for f in ("account_first", "account_more", "account_keys32", "nonce", "balance32", "storage_root32",
                                          "code_hash32", "slot_first", "slot_more", "slot_keys32", "slot_vals32")]


class Transition(C.Structure):
    _fields_ = [("n_nodes", C.c_uint64), ("nodes", C.c_void_p), ("node_off", C.c_void_p), ("nodes_bytes", C.c_uint64),
                ("n_blocks", C.c_uint64), ("pre_roots32", C.c_void_p), ("account_block", C.c_void_p)]


class RangeProofs(C.Structure):
    _fields_ = [("n_nodes", C.c_uint64), ("nodes", C.c_void_p), ("node_off", C.c_void_p), ("nodes_bytes", C.c_uint64),
                ("n_ranges", C.c_uint64), ("roots32", C.c_void_p), ("origin32", C.c_void_p), ("range_flags", C.c_void_p),
                ("entry_first", C.c_void_p), ("keys32", C.c_void_p), ("vals", C.c_void_p), ("val_off", C.c_void_p)]


RANGE_WHOLE = 1  # PHANT_GPU_RANGE_WHOLE: no boundary proof, the entries are the whole trie


ACCOUNT_DELETE = 1         # PHANT_GPU_ACCOUNT_DELETE: remove the account and all of its storage
ACCOUNT_CLEAR_STORAGE = 2  # PHANT_GPU_ACCOUNT_CLEAR_STORAGE: drop its storage before the diff's slots (re-created account)


EXPORTS = [
    "phant_gpu_abi_version", "phant_gpu_create", "phant_gpu_destroy", "phant_gpu_set_flags", "phant_gpu_set_stream", "phant_gpu_strerror",
    "phant_gpu_last_error", "phant_gpu_get_stats", "phant_gpu_reset_stats", "phant_gpu_synchronize",
    "phant_gpu_keccak256_batch", "phant_gpu_keccak256_batch_async", "phant_gpu_mpt_root", "phant_gpu_mpt_roots", "phant_gpu_state_root", "phant_gpu_state_subtree_roots", "phant_gpu_ecrecover_batch", "phant_gpu_verify_proofs", "phant_gpu_verify_witness",
    "phant_gpu_read_state",
    "phant_gpu_logs_bloom", "phant_gpu_trie_open", "phant_gpu_trie_root", "phant_gpu_trie_update", "phant_gpu_trie_close",
    "phant_gpu_resident_state_open", "phant_gpu_resident_state_apply", "phant_gpu_resident_state_root", "phant_gpu_resident_state_info",
    "phant_gpu_resident_state_close", "phant_gpu_resident_state_set_journal", "phant_gpu_resident_state_revert", "phant_gpu_resident_state_fork",
    "phant_gpu_resident_state_witness", "phant_gpu_resident_state_witness_copy", "phant_gpu_resident_state_prove",
    "phant_gpu_resident_state_prove_copy", "phant_gpu_resident_state_read", "phant_gpu_resident_state_range",
    "phant_gpu_resident_state_put_codes", "phant_gpu_resident_state_codes", "phant_gpu_resident_state_prune_codes",
    "phant_gpu_resident_state_trie_nodes", "phant_gpu_resident_state_trie_nodes_copy",
    "phant_gpu_resident_state_snap_ranges", "phant_gpu_resident_state_snap_ranges_copy",
    "phant_gpu_transition_roots", "phant_gpu_verify_ranges",
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
    L.phant_gpu_resident_state_fork.argtypes = [vp, C.c_uint32, C.POINTER(vp)]
    L.phant_gpu_resident_state_witness.argtypes = [vp, C.POINTER(StateDiff), C.POINTER(WitnessSize)]
    L.phant_gpu_resident_state_witness_copy.argtypes = [vp, vp, vp]
    L.phant_gpu_resident_state_prove.argtypes = [vp, C.POINTER(ProofRequest), C.POINTER(ProofSize)]
    L.phant_gpu_resident_state_prove_copy.argtypes = [vp, C.POINTER(Proofs)]
    L.phant_gpu_resident_state_read.argtypes = [vp, C.POINTER(ProofRequest), C.c_uint32, C.POINTER(StateReadValues), vp]
    L.phant_gpu_resident_state_range.argtypes = [vp, C.POINTER(RangeRequest), C.c_uint32, C.POINTER(RangeValues), vp]
    L.phant_gpu_resident_state_put_codes.argtypes = [vp, vp, vp, C.c_uint64, vp]
    L.phant_gpu_resident_state_codes.argtypes = [vp, vp, C.c_uint64, vp, vp, vp, C.c_uint64]
    L.phant_gpu_resident_state_prune_codes.argtypes = [vp]
    L.phant_gpu_resident_state_trie_nodes.argtypes = [vp, C.POINTER(TrieNodeRequest), C.POINTER(WitnessSize)]
    L.phant_gpu_resident_state_trie_nodes_copy.argtypes = [vp, C.POINTER(TrieNodes)]
    L.phant_gpu_resident_state_snap_ranges.argtypes = [vp, C.POINTER(SnapRequest), C.POINTER(SnapSize)]
    L.phant_gpu_resident_state_snap_ranges_copy.argtypes = [vp, C.POINTER(SnapRanges)]
    L.phant_gpu_transition_roots.argtypes = [vp, C.POINTER(Transition), C.POINTER(StateDiff), vp, vp, vp]
    L.phant_gpu_verify_ranges.argtypes = [vp, C.POINTER(RangeProofs), vp, vp]
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

    # G
    def verify_ranges(self, nodes, node_off, roots32, origin32, entry_first, keys32, vals, val_off, range_flags=None):
        """check n range-proof answers against their roots in one call (phant_gpu_verify_ranges): the boundary proofs' node
        set (CSR), per range its root and origin (n x 32) and flags (RANGE_WHOLE, or None), entry_first (n + 1) over the
        entries' hashed keys (32 bytes each) and leaf values (CSR).  Returns (status n: 1 accepted, 0 rejected, 3 a node
        missing; more n: 1 when an accepted range's trie holds a key above its last entry)."""
        off = np.ascontiguousarray(node_off, dtype=np.uint64)
        data = np.ascontiguousarray(nodes, dtype=np.uint8)
        roots = np.ascontiguousarray(roots32, dtype=np.uint8).reshape(-1)
        n = roots.size // 32
        org = _u8_rows(origin32, n, 32)
        first = np.ascontiguousarray(entry_first, dtype=np.uint64)
        ne = int(first[-1])
        keys = _u8_rows(keys32, ne, 32)
        vdata = np.ascontiguousarray(vals, dtype=np.uint8)
        voff = np.ascontiguousarray(val_off, dtype=np.uint64)
        fl = None if range_flags is None else np.ascontiguousarray(range_flags, dtype=np.uint8)
        rp = RangeProofs(len(off) - 1, _ptr(data), _ptr(off), int(off[-1]), n, _ptr(roots), _ptr(org), _ptr(fl), _ptr(first),
                         _ptr(keys) if ne else None, _ptr(vdata), _ptr(voff))
        status, more = np.zeros(max(n, 1), np.uint8), np.zeros(max(n, 1), np.uint8)
        self._chk(self.verify_ranges_raw(rp, status, more), "verify_ranges")
        return status[:n], more[:n]

    def verify_ranges_raw(self, rp, status, more=None):
        """a RangeProofs struct built by the caller (any pointers): the return code, not an exception"""
        return _lib().phant_gpu_verify_ranges(self._h, C.byref(rp), _ptr(status), _ptr(more))

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


def _csr_bytes(items):
    """byte strings -> (uint8 data, uint64 offsets), K's CSR layout"""
    off = np.zeros(len(items) + 1, np.uint64)
    off[1:] = np.cumsum([len(x) for x in items], dtype=np.uint64)
    data = np.frombuffer(b"".join(items) + bytes(1), np.uint8).copy()
    return data, off


def _u8_rows(a, n, width):
    a = np.ascontiguousarray(np.asarray(a, dtype=np.uint8)).reshape(-1)
    assert a.size == n * width, (a.size, n, width)
    return a


class ResidentState:
    """phant_gpu_resident_state: the account trie and every storage trie resident on the device (DESIGN.md §4.3c).
    apply() takes one block's changes with hashed keys; see StateDB-level helper phant_b200.host.ResidentStateDB."""

    def __init__(self, ctx, handle=None):
        """a new empty state on ctx, or (handle) the state a fork returned"""
        self.ctx = ctx
        self._h = handle
        if handle is None:
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

    @staticmethod
    def _request(account_keys32, slot_account=None, slot_keys32=None):
        ak = np.ascontiguousarray(np.asarray(account_keys32, dtype=np.uint8)).reshape(-1)
        assert ak.size % 32 == 0, ak.size
        n = ak.size // 32
        m = 0 if slot_account is None else len(slot_account)
        sa = None if not m else np.ascontiguousarray(slot_account, dtype=np.uint32)
        sk = None if not m else _u8_rows(slot_keys32, m, 32)
        q = ProofRequest(n, _ptr(ak) if n else None, m, _ptr(sa), _ptr(sk))
        q._keep = (ak, sa, sk)
        return q

    def prove(self, account_keys32, slot_account=None, slot_keys32=None):
        """account and storage proofs (eth_getProof) under the state as it is now (which is not changed): account_keys32 n x 32
        hashed addresses; slot_account (uint32, index into the accounts) and slot_keys32 (m x 32 hashed slots).  Returns a dict
        of numpy arrays: the node set (nodes, node_off), the chains (node_index, proof_first; proof p < n is account p, proof
        n + j slot j), roots32 and status (1 present, 2 absent) per proof, nonce / balance32 / storage_root32 / code_hash32 per
        account and slot_vals32 per slot."""
        q = self._request(account_keys32, slot_account, slot_keys32)
        size = ProofSize()
        self.ctx._chk(_lib().phant_gpu_resident_state_prove(self._h, C.byref(q), C.byref(size)), "resident_state_prove")
        n, m = q.n_accounts, q.n_slots
        r = dict(nodes=np.zeros(max(size.nodes_bytes, 1), np.uint8), node_off=np.zeros(size.n_nodes + 1, np.uint64),
                 node_index=np.zeros(max(size.n_refs, 1), np.uint64), proof_first=np.zeros(n + m + 1, np.uint64),
                 roots32=np.zeros((max(n + m, 1), 32), np.uint8), status=np.zeros(max(n + m, 1), np.uint8),
                 nonce=np.zeros(max(n, 1), np.uint64), balance32=np.zeros((max(n, 1), 32), np.uint8),
                 storage_root32=np.zeros((max(n, 1), 32), np.uint8), code_hash32=np.zeros((max(n, 1), 32), np.uint8),
                 slot_vals32=np.zeros((max(m, 1), 32), np.uint8))
        self.ctx._chk(_lib().phant_gpu_resident_state_prove_copy(self._h, C.byref(Proofs(*[_ptr(r[f]) for f, _ in Proofs._fields_]))),
                      "resident_state_prove_copy")
        r["nodes"], r["node_index"] = r["nodes"][:size.nodes_bytes], r["node_index"][:size.n_refs]
        for f, k in (("roots32", n + m), ("status", n + m), ("nonce", n), ("balance32", n), ("storage_root32", n), ("code_hash32", n),
                     ("slot_vals32", m)):
            r[f] = r[f][:k]
        return r

    def prove_raw(self, request):
        """a ProofRequest built by the caller: (return code, phant_gpu_proof_size)"""
        size = ProofSize()
        return _lib().phant_gpu_resident_state_prove(self._h, C.byref(request), C.byref(size)), size

    def prove_copy_raw(self, proofs):
        """a Proofs struct built by the caller: the return code"""
        return _lib().phant_gpu_resident_state_prove_copy(self._h, C.byref(proofs))

    def read(self, account_keys32, slot_account=None, slot_keys32=None, back=0):
        """account and slot values of the state as it is now (back = 0) or as it was `back` applies ago (the state revert(back)
        would return to), read without changing anything; keys as for prove(), repeats allowed.  Returns (dict of numpy
        arrays: account_status (1 present, 2 absent), nonce, balance32, storage_root32, code_hash32 per account, slot_status and
        slot_vals32 per slot; the root they belong to)."""
        q = self._request(account_keys32, slot_account, slot_keys32)
        n, m = q.n_accounts, q.n_slots
        r = dict(account_status=np.zeros(n, np.uint8), nonce=np.zeros(n, np.uint64), balance32=np.zeros((n, 32), np.uint8),
                 storage_root32=np.zeros((n, 32), np.uint8), code_hash32=np.zeros((n, 32), np.uint8), slot_status=np.zeros(m, np.uint8),
                 slot_vals32=np.zeros((m, 32), np.uint8))
        root = np.zeros(32, np.uint8)
        v = StateReadValues(*[_ptr(r[f]) if r[f].size else None for f, _ in StateReadValues._fields_])
        self.ctx._chk(_lib().phant_gpu_resident_state_read(self._h, C.byref(q), back, C.byref(v), _ptr(root)), "resident_state_read")
        return r, root.tobytes()

    def read_raw(self, request, back, values, root):
        """a ProofRequest and StateReadValues built by the caller (any pointers): the return code"""
        return _lib().phant_gpu_resident_state_read(self._h, C.byref(request), back, C.byref(values), _ptr(root))

    def range(self, account_ranges=(), storage_ranges=(), back=0):
        """account and storage ranges of the state as it is now (back = 0) or as it was `back` applies ago, read without
        changing anything.  account_ranges: [(origin32, limit32, max)]; storage_ranges: [(account key32, origin32, limit32,
        max)]; keys hashed, bounds inclusive.  Returns (dict of numpy arrays: account_first (n + 1), account_more (n),
        account_keys32 / nonce / balance32 / storage_root32 / code_hash32 per account entry, slot_first (m + 1), slot_more (m),
        slot_keys32 / slot_vals32 per slot entry; the root they belong to).  Range r's entries are
        [account_first[r], account_first[r + 1]) (slot_first for storage ranges).  Host buffers hold sum(max) entries, so a
        `max` of 2**32 - 1 wants that much host memory: ask in chunks."""
        cat = lambda xs: np.frombuffer(b"".join(xs), np.uint8).copy() if xs else np.zeros(32, np.uint8)  # noqa: E731
        n, m = len(account_ranges), len(storage_ranges)
        ao, al = cat([r[0] for r in account_ranges]), cat([r[1] for r in account_ranges])
        amax = np.array([r[2] for r in account_ranges] or [0], np.uint32)
        sa, so, sl = (cat([r[i] for r in storage_ranges]) for i in range(3))
        smax = np.array([r[3] for r in storage_ranges] or [0], np.uint32)
        q = RangeRequest(n, _ptr(ao), _ptr(al), _ptr(amax), m, _ptr(sa), _ptr(so), _ptr(sl), _ptr(smax))
        ea, es = int(amax[:n].sum()), int(smax[:m].sum())
        r = dict(account_first=np.zeros(n + 1, np.uint64), account_more=np.zeros(max(n, 1), np.uint8),
                 account_keys32=np.zeros((max(ea, 1), 32), np.uint8), nonce=np.zeros(max(ea, 1), np.uint64),
                 balance32=np.zeros((max(ea, 1), 32), np.uint8), storage_root32=np.zeros((max(ea, 1), 32), np.uint8),
                 code_hash32=np.zeros((max(ea, 1), 32), np.uint8), slot_first=np.zeros(m + 1, np.uint64),
                 slot_more=np.zeros(max(m, 1), np.uint8), slot_keys32=np.zeros((max(es, 1), 32), np.uint8),
                 slot_vals32=np.zeros((max(es, 1), 32), np.uint8))
        root = np.zeros(32, np.uint8)
        v = RangeValues(*[_ptr(r[f]) for f, _ in RangeValues._fields_])
        self.ctx._chk(_lib().phant_gpu_resident_state_range(self._h, C.byref(q), back, C.byref(v), _ptr(root)), "resident_state_range")
        ea, es = int(r["account_first"][n]), int(r["slot_first"][m])
        for f in ("account_keys32", "nonce", "balance32", "storage_root32", "code_hash32"):
            r[f] = r[f][:ea]
        r["slot_keys32"], r["slot_vals32"] = r["slot_keys32"][:es], r["slot_vals32"][:es]
        r["account_more"], r["slot_more"] = r["account_more"][:n], r["slot_more"][:m]
        return r, root.tobytes()

    def range_raw(self, request, back, values, root):
        """a RangeRequest and RangeValues built by the caller (any pointers): the return code"""
        return _lib().phant_gpu_resident_state_range(self._h, C.byref(request), back, C.byref(values), _ptr(root))

    def put_codes(self, codes):
        """store contract codes by keccak(code) beside the state (DESIGN.md §4.3i): codes is a list of bytes; each code the
        store does not hold is stored once, the empty code never.  Returns the hashes, n x 32 uint8, in the caller's order."""
        data, off = _csr_bytes(codes)
        hashes = np.zeros((max(len(codes), 1), 32), np.uint8)
        self.ctx._chk(self.put_codes_raw(data, off, len(codes), hashes), "resident_state_put_codes")
        return hashes[:len(codes)]

    def put_codes_raw(self, codes, code_off, n, hashes32):
        """any pointers: the return code"""
        return _lib().phant_gpu_resident_state_put_codes(self._h, _ptr(codes), _ptr(code_off), n, _ptr(hashes32))

    def codes(self, hashes32):
        """the codes behind n code hashes (n x 32 uint8, repeats allowed), read without changing anything: (status, [bytes]);
        status 1 held (keccak("") always, with b""), 2 not held (b"")"""
        h = np.ascontiguousarray(np.asarray(hashes32, dtype=np.uint8)).reshape(-1)
        assert h.size % 32 == 0, h.size
        n = h.size // 32
        status, off = np.zeros(max(n, 1), np.uint8), np.zeros(n + 1, np.uint64)
        self.ctx._chk(self.codes_raw(h, n, status, off, None, 0), "resident_state_codes")
        data = np.zeros(max(int(off[n]), 1), np.uint8)
        if off[n]:
            self.ctx._chk(self.codes_raw(h, n, status, off, data, data.size), "resident_state_codes")
        return status[:n], [data[int(off[i]):int(off[i + 1])].tobytes() for i in range(n)]

    def codes_raw(self, hashes32, n, status, code_off, codes, codes_cap):
        """any pointers: the return code"""
        return _lib().phant_gpu_resident_state_codes(self._h, _ptr(hashes32), n, _ptr(status), _ptr(code_off), _ptr(codes), codes_cap)

    def prune_codes(self):
        """drop every held code no account names at the current root or at a root the journal reaches"""
        self.ctx._chk(_lib().phant_gpu_resident_state_prune_codes(self._h), "resident_state_prune_codes")

    @staticmethod
    def _trie_node_request(paths, path_len, path_trie=None, storage_accounts=None):
        pl = np.ascontiguousarray(path_len, dtype=np.uint8).reshape(-1)
        n = pl.size
        pa = _u8_rows(paths, n, 32) if n else np.zeros(32, np.uint8)
        pt = None if path_trie is None else np.ascontiguousarray(path_trie, dtype=np.uint32).reshape(-1)
        sa = None if storage_accounts is None else np.ascontiguousarray(np.asarray(storage_accounts, dtype=np.uint8)).reshape(-1)
        m = 0 if sa is None else sa.size // 32
        q = TrieNodeRequest(n, _ptr(pa), _ptr(pl) if n else None, _ptr(pt) if n else None, m, _ptr(sa) if m else None)
        q._keep = (pa, pl, pt, sa)
        return q

    def trie_nodes(self, paths, path_len, path_trie=None, storage_accounts=None):
        """trie nodes by path (snap's GetTrieNodes, DESIGN.md §4.3k) of the state as it is now (which is not changed): paths
        n x 32 uint8 (nibble i of path p is nibble i of paths[p], high nibble first), path_len n nibble counts (0..64),
        path_trie n uint32 (0 the account trie, 1 + j the storage trie of storage_accounts[j]; None: all 0), storage_accounts
        m x 32 hashed addresses.  Returns (status, [bytes]): status 1 with the RLP of the node that starts at the path (the
        root, or a node its parent references by hash), 2 with b"" when there is none; in the caller's order."""
        q = self._trie_node_request(paths, path_len, path_trie, storage_accounts)
        rc, size = self.trie_nodes_raw(q)
        self.ctx._chk(rc, "resident_state_trie_nodes")
        n = q.n_paths
        status, off = np.zeros(max(n, 1), np.uint8), np.zeros(n + 1, np.uint64)
        data = np.zeros(max(size.nodes_bytes, 1), np.uint8)
        self.ctx._chk(self.trie_nodes_copy_raw(TrieNodes(_ptr(status), _ptr(off), _ptr(data))), "resident_state_trie_nodes_copy")
        return status[:n], [data[int(off[i]):int(off[i + 1])].tobytes() for i in range(n)]

    def trie_nodes_raw(self, request):
        """a TrieNodeRequest built by the caller: (return code, phant_gpu_witness_size)"""
        size = WitnessSize()
        return _lib().phant_gpu_resident_state_trie_nodes(self._h, C.byref(request), C.byref(size)), size

    def trie_nodes_copy_raw(self, out):
        """a TrieNodes struct built by the caller: the return code"""
        return _lib().phant_gpu_resident_state_trie_nodes_copy(self._h, C.byref(out))

    @staticmethod
    def _snap_request(account_requests=(), storage_requests=()):
        cat = lambda xs: np.frombuffer(b"".join(bytes(x) for x in xs), np.uint8).copy() if xs else np.zeros(32, np.uint8)  # noqa: E731
        n, m = len(account_requests), len(storage_requests)
        ao, al = cat([r[0] for r in account_requests]), cat([r[1] for r in account_requests])
        ab = np.array([r[2] for r in account_requests] or [0], np.uint64)
        first = np.zeros(m + 1, np.uint64)
        first[1:] = np.cumsum([len(r[0]) for r in storage_requests], dtype=np.uint64)
        sa = cat([a for r in storage_requests for a in r[0]])
        so, sl = cat([r[1] for r in storage_requests]), cat([r[2] for r in storage_requests])
        sb = np.array([r[3] for r in storage_requests] or [0], np.uint64)
        q = SnapRequest(n, _ptr(ao), _ptr(al), _ptr(ab), m, _ptr(first), _ptr(sa), _ptr(so), _ptr(sl), _ptr(sb))
        q._keep = (ao, al, ab, first, sa, so, sl, sb)
        return q

    def snap_ranges(self, account_requests=(), storage_requests=()):
        """the answers of snap GetAccountRange and GetStorageRanges requests (DESIGN.md §4.3m) of the state as it is now
        (which is not changed).  account_requests: [(origin32, limit32, bytes)]; storage_requests: [([account key32, ...],
        origin32, limit32, bytes)]; keys hashed.  Returns dict(accounts=[[(key, slim body)] per account request],
        slots=[[[(key, body)] per served account] per storage request], proofs=[[node bytes] per answer, account requests
        first], size=phant_gpu_snap_size as a dict)."""
        q = self._snap_request(account_requests, storage_requests)
        rc, size = self.snap_ranges_raw(q)
        self.ctx._chk(rc, "resident_state_snap_ranges")
        n, m = q.n_account_requests, q.n_storage_requests
        z = lambda k, t=np.uint64: np.zeros(max(int(k), 1), t)  # noqa: E731
        r = dict(account_first=z(n + 1), account_keys32=z(32 * size.n_accounts, np.uint8), account_body_off=z(size.n_accounts + 1),
                 account_bodies=z(size.account_bytes, np.uint8), served_first=z(m + 1), slot_first=z(size.n_served + 1),
                 slot_keys32=z(32 * size.n_slots, np.uint8), slot_body_off=z(size.n_slots + 1), slot_bodies=z(size.slot_bytes, np.uint8),
                 proof_first=z(n + m + 1), node_index=z(size.n_refs), nodes=z(size.nodes_bytes, np.uint8), node_off=z(size.n_nodes + 1))
        self.ctx._chk(self.snap_ranges_copy_raw(SnapRanges(*[_ptr(r[f]) for f, _ in SnapRanges._fields_])), "resident_state_snap_ranges_copy")
        blob = lambda data, off, i: data[int(off[i]):int(off[i + 1])].tobytes()  # noqa: E731
        key = lambda keys, e: keys[32 * e:32 * e + 32].tobytes()  # noqa: E731
        af, sf, slf, pf = r["account_first"], r["served_first"], r["slot_first"], r["proof_first"]
        accounts = [[(key(r["account_keys32"], e), blob(r["account_bodies"], r["account_body_off"], e)) for e in range(int(af[i]), int(af[i + 1]))]
                    for i in range(n)]
        slots = [[[(key(r["slot_keys32"], e), blob(r["slot_bodies"], r["slot_body_off"], e)) for e in range(int(slf[s]), int(slf[s + 1]))]
                  for s in range(int(sf[j]), int(sf[j + 1]))] for j in range(m)]
        proofs = [[blob(r["nodes"], r["node_off"], int(k)) for k in r["node_index"][int(pf[i]):int(pf[i + 1])]] for i in range(n + m)]
        return dict(accounts=accounts, slots=slots, proofs=proofs, size={f: getattr(size, f) for f, _ in SnapSize._fields_[:8]})

    def snap_ranges_raw(self, request):
        """a SnapRequest built by the caller: (return code, phant_gpu_snap_size)"""
        size = SnapSize()
        return _lib().phant_gpu_resident_state_snap_ranges(self._h, C.byref(request), C.byref(size)), size

    def snap_ranges_copy_raw(self, out):
        """a SnapRanges struct built by the caller: the return code"""
        return _lib().phant_gpu_resident_state_snap_ranges_copy(self._h, C.byref(out))

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
                "journal_bytes": i.journal_bytes, "n_codes": i.n_codes, "code_bytes": i.code_bytes}

    def set_journal(self, depth):
        """keep the undo records of the last `depth` successful applies on the device (0: none)"""
        self.ctx._chk(_lib().phant_gpu_resident_state_set_journal(self._h, depth), "resident_state_set_journal")

    def revert(self, n=1):
        """undo the last n successful applies, newest first; returns the root before the oldest of them"""
        out = np.zeros(32, np.uint8)
        self.ctx._chk(_lib().phant_gpu_resident_state_revert(self._h, n, _ptr(out)), "resident_state_revert")
        return out.tobytes()

    def fork(self, back=0):
        """a new, independent ResidentState holding exactly the state revert(back) would return to (back = 0: a copy of the
        state as it is now); this one is not changed.  Every call works on the fork at that root -- prove, trie_nodes,
        witness, read, range, and apply for a side branch (DESIGN.md §4.3l).  The fork starts with journal depth 0 and an
        empty code store, shares no device memory with this state, and is closed on its own."""
        h = C.c_void_p()
        self.ctx._chk(self.fork_raw(back, h), "resident_state_fork")
        return ResidentState(self.ctx, h)

    def fork_raw(self, back, out):
        """out: a c_void_p that receives the fork's handle, or None (a NULL out): the return code"""
        return _lib().phant_gpu_resident_state_fork(self._h, back, None if out is None else C.byref(out))

    def close(self):
        if getattr(self, "_h", None):
            _lib().phant_gpu_resident_state_close(self._h)
            self._h = None
        if self in getattr(self.ctx, "_tries", []):
            self.ctx._tries.remove(self)
