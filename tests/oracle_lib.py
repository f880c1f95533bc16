"""ctypes doorway to oracle/_build/liboracle.so -- the CPU checker (TEST INFRASTRUCTURE).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs import this.
"""
import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
LIB_PATH = os.path.join(ORACLE_DIR, "_build", "liboracle.so")
REF_KECCAK_PATH = os.path.join(ORACLE_DIR, "_ref", "libref_keccak.so")
REF_EVMONE_PATH = os.path.join(ORACLE_DIR, "_ref", "libref_evmone_mpt.so")

u8p = C.POINTER(C.c_uint8)
u32p = C.POINTER(C.c_uint32)
u64p = C.POINTER(C.c_uint64)


def build():
    """(re)build the oracle; also builds oracle/_ref when the reference checkout is present."""
    subprocess.run(["make", "-s", "-C", ORACLE_DIR], check=True, env={**os.environ, "CC": "gcc", "CXX": "g++"})


def _p(a, t):
    return a.ctypes.data_as(t) if a is not None else None


def _u8(b):
    return np.frombuffer(bytes(b), dtype=np.uint8) if not isinstance(b, np.ndarray) else b


def csr(items, off_dtype=np.uint64):
    """list of bytes -> (concatenated uint8 array, offsets)"""
    off = np.zeros(len(items) + 1, dtype=off_dtype)
    if items:
        off[1:] = np.cumsum([len(x) for x in items])
    data = np.frombuffer(b"".join(bytes(x) for x in items), dtype=np.uint8) if items else np.zeros(0, np.uint8)
    if data.size == 0:
        data = np.zeros(1, np.uint8)
    return np.ascontiguousarray(data), off


class Accounts(C.Structure):
    _fields_ = [("n_accounts", C.c_uint64), ("addr20", u8p), ("nonce", u64p), ("balance32", u8p), ("code", u8p),
                ("code_off", u64p), ("slot_keys32", u8p), ("slot_vals32", u8p), ("slot_off", u64p)]


class ProofBatch(C.Structure):
    _fields_ = [("n_proofs", C.c_uint64), ("nodes", u8p), ("node_off", u64p), ("proof_first", u64p), ("keys32", u8p),
                ("roots32", u8p), ("n_roots", C.c_uint64), ("node_index", u64p)]


KECCAK_FN = C.CFUNCTYPE(None, u8p, C.c_size_t, u8p)


class Oracle:
    def __init__(self):
        if not os.path.exists(LIB_PATH):
            build()
        self.lib = L = C.CDLL(LIB_PATH)
        L.oracle_keccak256.argtypes = [u8p, C.c_size_t, u8p]
        L.oracle_keccak256_batch.argtypes = [u8p, u64p, C.c_uint64, u8p, C.c_int]
        L.oracle_set_keccak.argtypes = [C.c_void_p]
        L.oracle_mptize.argtypes = [u8p, u32p, u8p, u64p, C.c_uint64, u8p]
        L.oracle_mptize.restype = C.c_int
        L.oracle_trie_build.argtypes = [u8p, u32p, u8p, u64p, C.c_uint64]
        L.oracle_trie_build.restype = C.c_void_p
        L.oracle_trie_root.argtypes = [C.c_void_p, u8p]
        L.oracle_trie_stats.argtypes = [C.c_void_p, u64p, u64p, u64p]
        L.oracle_trie_prove.argtypes = [C.c_void_p, u8p, C.c_uint32, u8p, C.c_uint64, u64p, C.c_uint32]
        L.oracle_trie_prove.restype = C.c_int
        L.oracle_trie_free.argtypes = [C.c_void_p]
        L.oracle_state_root.argtypes = [C.POINTER(Accounts), u8p]
        L.oracle_state_root.restype = C.c_int
        L.oracle_verify_proofs.argtypes = [C.POINTER(ProofBatch), u64p, u8p, u64p, u32p, C.c_int]
        L.oracle_ctrie_open.argtypes = [C.c_uint32, C.c_uint64]
        L.oracle_ctrie_open.restype = C.c_void_p
        L.oracle_ctrie_root.argtypes = [C.c_void_p, u8p]
        L.oracle_ctrie_update.argtypes = [C.c_void_p, u8p, u8p, u32p, C.c_uint64, u8p]
        L.oracle_ctrie_free.argtypes = [C.c_void_p]
        L.oracle_synth_c2_bytes_per_proof.argtypes = [C.c_uint32]
        L.oracle_synth_c2_bytes_per_proof.restype = C.c_uint64
        L.oracle_synth_c2.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint32, C.c_int, u8p, u64p, u64p, u8p, u8p, C.c_int]
        L.oracle_synth_c3_sizes.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, u32p, u32p]
        L.oracle_synth_c3.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.c_int, u8p, u64p, u64p, u8p, u8p, C.c_int]
        self._ref = None

    # -- reference keccak plug (oracle/_ref) --
    def use_reference_keccak(self, on=True):
        """Route every oracle hash through the reference's own compiled keccak.c (oracle/_ref)."""
        if not on:
            self.lib.oracle_set_keccak(None)
            return True
        if not os.path.exists(REF_KECCAK_PATH):
            return False
        if self._ref is None:
            self._ref = C.CDLL(REF_KECCAK_PATH)

            class H256(C.Structure):
                _fields_ = [("b", C.c_uint8 * 32)]
            self._ref.ethash_keccak256.argtypes = [u8p, C.c_size_t]
            self._ref.ethash_keccak256.restype = H256
        self.lib.oracle_use_ref_keccak.argtypes = [C.c_char_p]
        self.lib.oracle_use_ref_keccak.restype = C.c_int
        if self.lib.oracle_use_ref_keccak(REF_KECCAK_PATH.encode()) != 0:
            return False
        return True

    def ref_keccak256(self, data):
        if self._ref is None:
            self.use_reference_keccak(True)
            self.lib.oracle_set_keccak(None)
        a = _u8(data) if len(data) else np.zeros(1, np.uint8)
        h = self._ref.ethash_keccak256(_p(a, u8p), len(data))
        return bytes(h.b)

    # -- keccak --
    def keccak256(self, data):
        a = _u8(data) if len(data) else np.zeros(1, np.uint8)
        out = np.zeros(32, np.uint8)
        self.lib.oracle_keccak256(_p(a, u8p), len(data), _p(out, u8p))
        return out.tobytes()

    def keccak256_batch(self, msgs, off, threads=1):
        n = len(off) - 1
        out = np.zeros((n, 32), np.uint8)
        self.lib.oracle_keccak256_batch(_p(msgs, u8p), _p(off, u64p), n, _p(out, u8p), threads)
        return out

    def logs_bloom(self, items, owner, n_blooms):
        data, off = csr(items)
        own = np.array(owner or [0], np.uint32)
        out = np.zeros((max(n_blooms, 1), 256), np.uint8)
        self.lib.oracle_logs_bloom.argtypes = [u8p, u64p, u32p, C.c_uint64, C.c_uint64, u8p]
        self.lib.oracle_logs_bloom(_p(data, u8p), _p(off, u64p), _p(own, u32p), len(items), n_blooms, _p(out, u8p))
        return out[:n_blooms]

    # -- secp256k1 recovery --
    def ecrecover(self, hash32, sig65):
        """-> 65-byte public key (0x04 || X || Y) or None when the signature recovers no key"""
        out = C.create_string_buffer(65)
        self.lib.oracle_ecrecover.restype = C.c_int
        rc = self.lib.oracle_ecrecover(bytes(hash32), bytes(sig65), out)
        return out.raw if rc == 0 else None

    def secp256k1_pubkey(self, priv32):
        out = C.create_string_buffer(65)
        assert self.lib.oracle_secp256k1_pubkey(bytes(priv32), out) == 0
        return out.raw

    # -- mptize --
    def mptize(self, kv):
        keys, koff = csr([k for k, _ in kv], np.uint32)
        vals, voff = csr([v for _, v in kv], np.uint64)
        return self.mptize_csr(keys, koff, vals, voff)

    def mptize_csr(self, keys, key_off, vals, val_off):
        """the same root from CSR arrays (keys uint8 + uint32 offsets, values uint8 + uint64 offsets), for key sets too large
        for a Python list of pairs"""
        n = len(key_off) - 1
        assert len(val_off) == n + 1 and key_off.dtype == np.uint32 and val_off.dtype == np.uint64
        keys = np.ascontiguousarray(keys if keys.size else np.zeros(1, np.uint8)).reshape(-1)
        vals = np.ascontiguousarray(vals if vals.size else np.zeros(1, np.uint8)).reshape(-1)
        key_off, val_off = np.ascontiguousarray(key_off), np.ascontiguousarray(val_off)
        out = np.zeros(32, np.uint8)
        rc = self.lib.oracle_mptize(_p(keys, u8p), _p(key_off, u32p), _p(vals, u8p), _p(val_off, u64p), n, _p(out, u8p))
        if rc != 0:
            raise ValueError("keys not strictly sorted")
        return out.tobytes()

    def trie(self, kv):
        return Trie(self, kv)

    # -- state root --
    def state_root(self, accounts):
        """accounts: list of dict(address hex20, nonce int, balance hex32, code hex, storage {hex32: hex32})"""
        n = len(accounts)
        addr = np.frombuffer(b"".join(bytes.fromhex(a["address"]) for a in accounts), np.uint8) if n else np.zeros(1, np.uint8)
        nonce = np.array([a["nonce"] for a in accounts], np.uint64) if n else np.zeros(1, np.uint64)
        bal = np.frombuffer(b"".join(bytes.fromhex(a["balance"]) for a in accounts), np.uint8) if n else np.zeros(1, np.uint8)
        code, coff = csr([bytes.fromhex(a["code"]) for a in accounts])
        sk, sv, soff = [], [], [0]
        for a in accounts:
            for k, v in a["storage"].items():
                sk.append(bytes.fromhex(k))
                sv.append(bytes.fromhex(v))
            soff.append(len(sk))
        skeys = np.frombuffer(b"".join(sk), np.uint8) if sk else np.zeros(1, np.uint8)
        svals = np.frombuffer(b"".join(sv), np.uint8) if sv else np.zeros(1, np.uint8)
        soff = np.array(soff, np.uint64)
        keep = (addr, nonce, bal, code, coff, skeys, svals, soff)
        st = Accounts(n, _p(addr, u8p), _p(nonce, u64p), _p(bal, u8p), _p(code, u8p), _p(coff, u64p), _p(skeys, u8p),
                      _p(svals, u8p), _p(soff, u64p))
        out = np.zeros(32, np.uint8)
        rc = self.lib.oracle_state_root(C.byref(st), _p(out, u8p))
        assert rc == 0
        del keep
        return out.tobytes()

    # -- proofs --
    def verify_proofs(self, nodes, node_off, proof_first, keys32, roots32, threads=1, node_index=None):
        n = len(proof_first) - 1
        n_roots = roots32.size // 32
        nodes = np.ascontiguousarray(nodes)
        b = ProofBatch(n, _p(nodes, u8p), _p(node_off, u64p), _p(proof_first, u64p), _p(keys32, u8p), _p(roots32, u8p), n_roots,
                       _p(node_index, u64p))
        bitmap = np.zeros((n + 63) // 64, np.uint64)
        status = np.zeros(max(n, 1), np.uint8)
        voff = np.zeros(max(n, 1), np.uint64)
        vlen = np.zeros(max(n, 1), np.uint32)
        self.lib.oracle_verify_proofs(C.byref(b), _p(bitmap, u64p), _p(status, u8p), _p(voff, u64p), _p(vlen, u32p), threads)
        return bitmap, status[:n], voff[:n], vlen[:n]

    def verify_bag(self, nodes, node_off, keys32, roots32, threads=1):
        n_nodes, n_keys = len(node_off) - 1, keys32.size // 32
        status = np.zeros(max(n_keys, 1), np.uint8)
        voff = np.zeros(max(n_keys, 1), np.uint64)
        vlen = np.zeros(max(n_keys, 1), np.uint32)
        self.lib.oracle_verify_bag.argtypes = [u8p, u64p, C.c_uint64, u8p, C.c_uint64, u8p, C.c_uint64, u8p, u64p, u32p, C.c_int]
        self.lib.oracle_verify_bag(_p(np.ascontiguousarray(nodes), u8p), _p(node_off, u64p), n_nodes, _p(keys32, u8p), n_keys, _p(roots32, u8p),
                                   roots32.size // 32, _p(status, u8p), _p(voff, u64p), _p(vlen, u32p), threads)
        return status[:n_keys], voff[:n_keys], vlen[:n_keys]

    # -- synthetic --
    def synth_c2(self, n, depth=8, first=0, corrupt=True, seed=0x5048414E54, threads=8):
        per = self.lib.oracle_synth_c2_bytes_per_proof(depth)
        nodes = np.zeros(n * per + 16, np.uint8)
        node_off = np.zeros(n * depth + 1, np.uint64)
        first_arr = np.zeros(n + 1, np.uint64)
        keys = np.zeros(n * 32, np.uint8)
        roots = np.zeros(n * 32, np.uint8)
        self.lib.oracle_synth_c2(seed, first, n, depth, int(corrupt), _p(nodes, u8p), _p(node_off, u64p), _p(first_arr, u64p),
                                 _p(keys, u8p), _p(roots, u8p), threads)
        return nodes, node_off, first_arr, keys, roots

    def synth_c3(self, n, first=0, corrupt=True, seed=0x5048414E54, threads=8):
        nn = np.zeros(n, np.uint32)
        nb = np.zeros(n, np.uint32)
        self.lib.oracle_synth_c3_sizes(seed, first, n, _p(nn, u32p), _p(nb, u32p))
        nodes = np.zeros(int(nb.sum()) + 16, np.uint8)
        node_off = np.zeros(int(nn.sum()) + 1, np.uint64)
        first_arr = np.zeros(n + 1, np.uint64)
        keys = np.zeros(n * 32, np.uint8)
        roots = np.zeros(n * 32, np.uint8)
        self.lib.oracle_synth_c3(seed, first, n, int(corrupt), _p(nodes, u8p), _p(node_off, u64p), _p(first_arr, u64p),
                                 _p(keys, u8p), _p(roots, u8p), threads)
        return nodes, node_off, first_arr, keys, roots

    def synth_blocks(self, n_blocks, txs=300, first=0, seed=0x5048414E54, threads=8):
        """C5: deduplicated block witnesses -> dict of numpy arrays (copies; the C buffers are freed)"""
        L = self.lib
        L.oracle_synth_blocks.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, C.c_int] + [C.POINTER(C.c_void_p)] * 7 + [u64p]
        L.oracle_free.argtypes = [C.c_void_p]
        ptrs = [C.c_void_p() for _ in range(7)]
        totals = (C.c_uint64 * 4)()
        L.oracle_synth_blocks(seed, first, n_blocks, txs, threads, *[C.byref(p) for p in ptrs], totals)
        tn, tb, ti, tp = (int(x) for x in totals)

        def take(p, dtype, count):
            a = np.ctypeslib.as_array(C.cast(p, C.POINTER(np.ctypeslib.as_ctypes_type(dtype))), shape=(count,)).copy()
            L.oracle_free(p)
            return a
        return dict(nodes=np.concatenate([take(ptrs[0], np.uint8, tb + 64)]), node_off=take(ptrs[1], np.uint64, tn + 1),
                    node_index=take(ptrs[2], np.uint64, ti + 1)[:ti], proof_first=take(ptrs[3], np.uint64, tp + 1),
                    keys32=take(ptrs[4], np.uint8, 32 * tp + 32)[:32 * tp], roots32=take(ptrs[5], np.uint8, 32 * tp + 32)[:32 * tp],
                    block_of_proof=take(ptrs[6], np.uint32, tp + 1)[:tp], n_nodes=tn, n_bytes=tb, n_refs=ti, n_proofs=tp)

    # -- complete trie --
    def ctrie(self, depth, seed=0x5048414E54):
        return CTrie(self, depth, seed)


class Trie:
    def __init__(self, o, kv):
        self.o = o
        keys, koff = csr([k for k, _ in kv], np.uint32)
        vals, voff = csr([v for _, v in kv], np.uint64)
        self.h = o.lib.oracle_trie_build(_p(keys, u8p), _p(koff, u32p), _p(vals, u8p), _p(voff, u64p), len(kv))
        if not self.h:
            raise ValueError("keys not strictly sorted")

    def root(self):
        out = np.zeros(32, np.uint8)
        self.o.lib.oracle_trie_root(self.h, _p(out, u8p))
        return out.tobytes()

    def stats(self):
        a, b, c = C.c_uint64(), C.c_uint64(), C.c_uint64()
        self.o.lib.oracle_trie_stats(self.h, C.byref(a), C.byref(b), C.byref(c))
        return a.value, b.value, c.value

    def prove(self, key):
        buf = np.zeros(1 << 20, np.uint8)
        off = np.zeros(130, np.uint64)
        k = _u8(key) if len(key) else np.zeros(1, np.uint8)
        n = self.o.lib.oracle_trie_prove(self.h, _p(k, u8p), len(key), _p(buf, u8p), buf.size, _p(off, u64p), 129)
        assert n >= 0
        return [buf[int(off[i]):int(off[i + 1])].tobytes() for i in range(n)]

    def __del__(self):
        if getattr(self, "h", None):
            self.o.lib.oracle_trie_free(self.h)
            self.h = None


class CTrie:
    def __init__(self, o, depth, seed):
        self.o = o
        self.h = o.lib.oracle_ctrie_open(depth, seed)

    def root(self):
        out = np.zeros(32, np.uint8)
        self.o.lib.oracle_ctrie_root(self.h, _p(out, u8p))
        return out.tobytes()

    def update(self, keys32, vals):
        v, voff = csr(vals, np.uint32)
        out = np.zeros(32, np.uint8)
        k = np.ascontiguousarray(keys32)
        self.o.lib.oracle_ctrie_update(self.h, _p(k, u8p), _p(v, u8p), _p(voff, u32p), len(vals), _p(out, u8p))
        return out.tobytes()

    def __del__(self):
        if getattr(self, "h", None):
            self.o.lib.oracle_ctrie_free(self.h)
            self.h = None


_singleton = None


def get():
    global _singleton
    if _singleton is None:
        _singleton = Oracle()
    return _singleton
