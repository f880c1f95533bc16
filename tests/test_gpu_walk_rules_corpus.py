"""The proof walk's decoding rules (R2-R4) on every device path, on malformed nodes whose hashes still match
(tests/walk_corpus.py): chain-form verify through the fused kernel, the two-kernel walk with the staged, direct and warp
Keccak kernels and without regrouping, in host- and device-pointer mode, under and over the 4,096 proofs where regrouping
starts; deduplicated chains; node sets (complete and with the malformed node missing); and pre-state reads with the
malformed node in the account trie and inside a storage trie.  Every result must equal the oracle bit for bit: status,
accept bitmap, value offset and length."""
import numpy as np
import pytest

import oracle_lib
import walk_corpus as wc
from helpers import rlp_list, rlp_str
from state_read_oracle import read_state
from test_oracle_proofs import batch_of

pytestmark = pytest.mark.gpu

FIELDS = ("account_status", "nonce", "balance32", "storage_root32", "code_hash32", "code_index", "slot_status", "slot_vals32")


@pytest.fixture(scope="module")
def ctx():
    from phant_b200 import gpu
    c = gpu.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def corpus(oracle):
    return wc.build(oracle.keccak256)


def tiled(corpus, n_min):
    """the corpus repeated until it has n_min proofs; it ends on a 16-byte boundary, so every node keeps its start residue"""
    reps = -(-n_min // len(corpus))
    return corpus * reps


def assert_verify_same(got, want, what):
    bitmap, status, voff, vlen = got
    bad = np.nonzero(status != want[1])[0]
    assert bad.size == 0, (what, bad[:10], status[bad[:10]], want[1][bad[:10]])
    assert (bitmap == want[0]).all(), what
    ok = want[1] == 1
    assert (voff[ok] == want[2][ok]).all() and (vlen[ok] == want[3][ok]).all(), what


def host_verify(ctx, nodes, node_off, first, keys, roots, flags, **kw):
    n = len(first) - 1
    out = (np.zeros((n + 63) // 64, np.uint64), np.full(n, 77, np.uint8), np.zeros(n, np.uint64), np.zeros(n, np.uint32))
    ctx.set_flags(flags)
    try:
        ctx.verify_proofs(n, np.ascontiguousarray(nodes), node_off, first, np.ascontiguousarray(keys), np.ascontiguousarray(roots),
                          roots.size // 32, *out, **kw)
    finally:
        ctx.set_flags(0)
    return out


def device_verify(ctx, nodes, node_off, first, keys, roots, flags):
    import torch
    from phant_b200 import gpu
    n = len(first) - 1
    dev = lambda a: torch.from_numpy(np.array(a)).cuda()  # noqa: E731
    d_nodes = dev(np.concatenate([nodes, np.zeros(64, np.uint8)]))
    d_off, d_first = dev(node_off.astype(np.int64)), dev(first.astype(np.int64))
    d_keys, d_roots = dev(keys), dev(roots)
    d_bitmap = torch.zeros((n + 63) // 64, dtype=torch.int64, device="cuda")
    d_status = torch.full((n,), 77, dtype=torch.uint8, device="cuda")
    d_voff = torch.zeros(n, dtype=torch.int64, device="cuda")
    d_vlen = torch.zeros(n, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    ctx.set_flags(gpu.FLAG_DEVICE_PTRS | flags)
    try:
        ctx.verify_proofs(n, d_nodes, d_off, d_first, d_keys, d_roots, roots.size // 32, d_bitmap, d_status, d_voff, d_vlen,
                          n_nodes=len(node_off) - 1, nodes_bytes=int(node_off[-1]))
        ctx.synchronize()
    finally:
        ctx.set_flags(0)
    return (d_bitmap.cpu().numpy().view(np.uint64), d_status.cpu().numpy(), d_voff.cpu().numpy().view(np.uint64),
            d_vlen.cpu().numpy().view(np.uint32))


@pytest.mark.parametrize("size", ["small", "tiled"])
def test_verify_every_path(ctx, oracle, corpus, size):
    """flags 0 (fused), unfused, direct, warp and no-binning, host and device pointers; the fused path reports the Keccak
    work of every node, also of the nodes a rejected proof never hashed"""
    from phant_b200 import gpu
    cases = corpus[:4000] if size == "small" else tiled(corpus, 4096 * 3)  # the first 4,000 hold every named case
    assert (len(cases) < 4096) == (size == "small")
    b = batch_of([c.proof() for c in cases])
    want = oracle.verify_proofs(*b, threads=8)
    for flags in (0, gpu.FLAG_UNFUSED_WALK, gpu.FLAG_KECCAK_DIRECT, gpu.FLAG_KECCAK_WARP, gpu.FLAG_NO_BINNING):
        ctx.reset_stats()
        assert_verify_same(host_verify(ctx, *b, flags), want, ("host", flags))
        if flags == 0:
            perms = int((np.diff(b[1].astype(np.int64)) // 136 + 1).sum())
            assert ctx.stats()["keccak_perms"] == perms
        assert_verify_same(device_verify(ctx, *b, flags), want, ("device", flags))


def test_verify_solo_leaves(ctx, oracle, corpus):
    """depth-0 leaf cases alone, so the leaf starts the node buffer (its path compared nibble by nibble, not with the wide
    load), fused and unfused"""
    from phant_b200 import gpu
    solo = [c for c in corpus if "/d0/" in c.name and c.name.startswith(("leaf/", "residue/leaf_136_at_0", "size/leaf"))]
    assert len(solo) > 60
    for c in solo:
        b = batch_of([c.proof()])
        want = oracle.verify_proofs(*b)
        assert int(want[1][0]) == c.status, c.name
        for flags in (0, gpu.FLAG_UNFUSED_WALK):
            assert_verify_same(host_verify(ctx, *b, flags), want, (c.name, flags))


def test_deduplicated_chains(ctx, oracle, corpus):
    """the tiled corpus as a deduplicated witness: every malformed node is shared by several proofs (staged and direct
    Keccak kernels; a deduplicated batch always takes the two-kernel walk)"""
    from phant_b200 import gpu
    cases = tiled(corpus, 4096 * 2)
    flat = [nd for c in cases for nd in c.nodes]
    uniq = list({nd: 1 for nd in flat})
    where = {nd: j for j, nd in enumerate(uniq)}
    unodes, uoff = oracle_lib.csr(uniq, np.uint64)
    index = np.array([where[nd] for nd in flat], np.uint64)
    _, _, first, keys, roots = batch_of([c.proof() for c in cases])
    want = oracle.verify_proofs(unodes, uoff, first, keys, roots, threads=8, node_index=index)
    for flags in (0, gpu.FLAG_KECCAK_DIRECT):
        got = host_verify(ctx, unodes, uoff, first, keys, roots, flags, node_index=index, n_nodes=len(uniq), nodes_bytes=int(uoff[-1]))
        assert_verify_same(got, want, ("dedup", flags))


def test_witness_bags(ctx, oracle, corpus):
    """every case's nodes in one node set (a root per key), complete and with each case's malformed node left out"""
    _, _, _, keys, roots = batch_of([c.proof() for c in corpus])
    n = len(corpus)
    for leave_out in (False, True):
        drop = {c.nodes[c.target] for c in corpus if leave_out and c.target is not None and c.name != "spacer"}
        bag = list({nd: 1 for c in corpus for nd in c.nodes if nd not in drop})
        bnodes, boff = oracle_lib.csr(bag, np.uint64)
        want = oracle.verify_bag(bnodes, boff, keys, roots, threads=8)
        st, vo, vl = np.full(n, 77, np.uint8), np.zeros(n, np.uint64), np.zeros(n, np.uint32)
        bitmap = np.zeros((n + 63) // 64, np.uint64)
        ctx.verify_witness(len(bag), np.concatenate([bnodes, np.zeros(64, np.uint8)]), boff, n, keys, roots, n, bitmap, st, vo, vl)
        assert (st == want[0]).all(), (leave_out, np.nonzero(st != want[0])[0][:10])
        ok = st == 1
        assert (vo[ok] == want[1][ok]).all() and (vl[ok] == want[2][ok]).all()
        if leave_out:
            reach = np.array([c.target is not None and c.name != "spacer" for c in corpus])
            assert (st[reach] == wc.MISSING).all()


def test_read_state(ctx, oracle, corpus):
    """P with the malformed node in the account trie (each case read as an account), and inside a storage trie: each case's
    root is the storage root of an account leaf, so the case is resealed through the account trie"""
    cases = [c for c in corpus if c.name != "spacer"]
    rng = np.random.default_rng(8)
    # storage: one account per case, its storage root the case's root, the slot key the case's key
    sel = cases[::3]
    addr_keys = sorted({rng.integers(0, 256, 32, dtype=np.uint8).tobytes() for _ in range(len(sel))})[:len(sel)]
    assert len(addr_keys) == len(sel)
    items = [(k, rlp_list([rlp_str(b"\x01"), rlp_str(b"\x02\x03"), rlp_str(c.root), rlp_str(oracle.keccak256(b""))]))
             for k, c in zip(addr_keys, sel)]
    trie = oracle.trie(items)
    aroot = trie.root()
    node_list = list({nd: 1 for k, _ in items for nd in trie.prove(k)})
    node_list += [nd for c in cases for nd in c.nodes]
    node_list = list({nd: 1 for nd in node_list})
    nodes, off = oracle_lib.csr(node_list, np.uint64)
    nodes = np.concatenate([nodes, np.zeros(64, np.uint8)])
    # accounts: the storage-trie holders (under the account root) and every case read as an account (under its own root)
    akeys = np.frombuffer(b"".join(k for k, _ in items) + b"".join(c.key for c in cases), np.uint8).copy()
    aroots = np.frombuffer(aroot * len(items) + b"".join(c.root for c in cases), np.uint8).copy()
    skeys = np.frombuffer(b"".join(c.key for c in sel), np.uint8).copy()
    sacc = np.arange(len(sel), dtype=np.uint32)
    na, ns = akeys.size // 32, skeys.size // 32
    out = dict(account_status=np.full(na, 0x77, np.uint8), nonce=np.full(na, 0x77, np.uint64), balance32=np.full((na, 32), 0x77, np.uint8),
               storage_root32=np.full((na, 32), 0x77, np.uint8), code_hash32=np.full((na, 32), 0x77, np.uint8),
               code_index=np.full(na, 0x77, np.uint32), slot_status=np.full(ns, 0x77, np.uint8), slot_vals32=np.full((ns, 32), 0x77, np.uint8))
    ctx.read_state(len(node_list), nodes, off, na, akeys, aroots, na, ns, skeys, sacc, 0, None, None, **out)
    want = read_state(oracle, nodes, off, aroots, akeys, skeys, sacc)
    for k in FIELDS:
        assert (np.asarray(out[k]) == np.asarray(want[k])).all(), (k, np.nonzero(np.asarray(out[k]) != np.asarray(want[k]))[0][:10])
    assert (out["account_status"][:len(items)] == 1).all()
    assert {0, 2} <= set(out["slot_status"].tolist())
