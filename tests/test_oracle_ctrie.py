"""The complete-trie oracle (oracle/ctrie.c) against a root recomputed in plain Python, at every RLP length edge of a leaf,
including leaves far larger than a stack buffer.  CPU only: the GPU resident-trie tests trust this oracle."""
import numpy as np

from helpers import _hp, rlp_list, rlp_str


def _nibbles(key):
    return [x for b in key for x in (b >> 4, b & 15)]


def test_ctrie_depth1_all_leaves_any_value_length(oracle):
    """depth 1: all 16 leaves rewritten in one update, so the root depends on no PRNG leaf; value lengths cover the empty
    value, the single byte below and at 0x80, the 55/56 string header edge, the 1-byte / 2-byte length edge at 256, and values
    of 2,020 and 5,000 bytes"""
    rng = np.random.default_rng(11)
    lengths = [0, 1, 1, 55, 56, 255, 256, 2020, 5000, 0, 1, 56, 256, 5000, 2020, 55]
    keys = rng.integers(0, 256, (16, 32), dtype=np.uint8)
    keys[:, 0] = (np.arange(16, dtype=np.uint8) << 4) | (keys[:, 0] & 15)   # leaf i sits at position i
    vals = [rng.integers(0, 256, n, dtype=np.uint8).tobytes() for n in lengths]
    vals[1], vals[2] = b"\x7f", b"\x80"                                   # one byte that encodes as itself, one that does not
    vals[10] = b"\x00"
    o = oracle.ctrie(1)
    root = o.update(np.ascontiguousarray(keys.reshape(-1)), vals)

    children = []
    for k, v in zip(keys, vals):
        leaf = rlp_list([rlp_str(_hp(_nibbles(k.tobytes())[1:], True)), rlp_str(v)])
        children.append(rlp_str(oracle.keccak256(leaf)))
    branch = rlp_list(children + [rlp_str(b"")])
    assert len(branch) == 532
    assert root == oracle.keccak256(branch)
    assert o.root() == root


def test_mptize_csr_matches_mptize(oracle):
    """the CSR entry point (used where the key set is too large for a list of pairs) gives the list entry point's roots"""
    rng = np.random.default_rng(13)
    for n in (0, 1, 2, 17, 3000):
        keys = np.unique(rng.integers(0, 256, (n, 32), dtype=np.uint8), axis=0)
        lens = rng.integers(0, 300, len(keys))
        kv = [(k.tobytes(), rng.integers(0, 256, int(l), dtype=np.uint8).tobytes()) for k, l in zip(keys, lens)]
        koff = (np.arange(len(kv) + 1) * 32).astype(np.uint32)
        voff = np.zeros(len(kv) + 1, np.uint64)
        voff[1:] = np.cumsum([len(v) for _, v in kv])
        vals = np.frombuffer(b"".join(v for _, v in kv), np.uint8)
        assert oracle.mptize_csr(keys.reshape(-1), koff, vals, voff) == oracle.mptize(kv), n


def test_ctrie_untouched_leaves_keep_their_prng_hash(oracle):
    """one leaf rewritten with a 3,000-byte value at depth 2: its sibling hashes are the open-time ones, so only the
    touched path changes; the same update applied twice gives the same root"""
    rng = np.random.default_rng(12)
    o = oracle.ctrie(2)
    r0 = o.root()
    key = rng.integers(0, 256, 32, dtype=np.uint8)
    val = rng.integers(0, 256, 3000, dtype=np.uint8).tobytes()
    r1 = o.update(np.ascontiguousarray(key), [val])
    assert r1 != r0
    assert o.update(np.ascontiguousarray(key), [val]) == r1
