#!/usr/bin/env python3
"""Call each trie builder entry point once on seeded inputs and print every result followed by the context's counters.
Run it against two builds of libphantgpu.so and diff the outputs: a host-side change (how scratch areas are sized and laid
out, say) must leave every result, launch count, copy size and Keccak message count as it was.  The world state's calls
and the node-set calls (W, P, T, G) print their return codes too, refusals included, and the world state's witness, proofs,
trie nodes and snap range answers are called in every order of the one result a state holds, and on a fork.  The
stateless calls (K, V, W, P, B, sender recovery, block reject counts) run with host and with device pointers, with each
nullable output left out, and with one refusal each.
  python tools/trie_calls.py [path/to/libphantgpu.so] > trie_calls_<tag>.txt
The trie builders run on every path: M's single-CTA and level-by-level BFS, both arena layouts, the leaf-reference cache,
the export, and kind 0's and kind 1's refusals and depth changes.
The library reads PHANT_GPU_CHUNK_MB once per process: run the script a second time with PHANT_GPU_CHUNK_MB=1 so that the
chain-form proof batch crosses in several chunks, and diff that run too.
Needs a GPU.
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from phant_b200 import gpu, host  # noqa: E402

if len(sys.argv) > 1:
    gpu.LIB_PATH = os.path.abspath(sys.argv[1])

import oracle_lib  # noqa: E402
from range_proof_corpus import accept_cases, mutations, random_tries  # noqa: E402
from resident_state_model import CLEAR, DELETE, Diff  # noqa: E402
from test_transition_model import random_case  # noqa: E402
from transition_oracle import EMPTY_ROOT, witness  # noqa: E402

COUNTERS = ("launches", "h2d_bytes", "d2h_bytes", "keccak_msgs", "keccak_bytes", "keccak_perms")


def show(ctx, name, result):
    st = ctx.stats()
    print(name, result, " ".join(f"{k}={st[k]}" for k in COUNTERS), flush=True)
    ctx.reset_stats()


def hexs(x):
    if isinstance(x, (bytes, bytearray)):
        return x.hex()
    if isinstance(x, np.ndarray):
        return x.tobytes().hex()
    return " ".join(hexs(e) for e in x)


def csr(items, off_dtype):
    off = np.zeros(len(items) + 1, off_dtype)
    off[1:] = np.cumsum([len(x) for x in items])
    return np.frombuffer(b"".join(items), np.uint8).copy() if items else np.zeros(1, np.uint8), off


def rbytes(rng, n):
    return bytes(rng.integers(0, 256, n, dtype=np.uint8))


def mpt_inputs(rng, n, key_len):
    keys = sorted({rbytes(rng, int(rng.integers(1, key_len + 1))) for _ in range(n)})
    vals = [rbytes(rng, int(rng.integers(1, 120))) for _ in keys]
    k, ko = csr(keys, np.uint32)
    v, vo = csr(vals, np.uint64)
    return k, ko, v, vo, len(keys)


def accounts(rng, n, slots_every=3, n_slots=20):
    addr = rng.integers(0, 256, (n, 20), dtype=np.uint8)
    nonce = rng.integers(0, 1000, n, dtype=np.uint64)
    bal = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    codes = [rbytes(rng, int(rng.integers(0, 300))) if i % 4 == 0 else b"" for i in range(n)]
    code, code_off = csr(codes, np.uint64)
    per = [n_slots if i % slots_every == 0 else 0 for i in range(n)]
    slot_off = np.zeros(n + 1, np.uint64)
    slot_off[1:] = np.cumsum(per)
    ns = int(slot_off[-1])
    sk = rng.integers(0, 256, (max(ns, 1), 32), dtype=np.uint8)
    sv = rng.integers(0, 256, (max(ns, 1), 32), dtype=np.uint8)
    sv[::5] = 0  # zero slots are dropped
    return n, addr, nonce, bal, code, code_off, sk, sv, slot_off


def digest(*arrays):
    return hashlib.sha256(b"".join(np.ascontiguousarray(a).tobytes() for a in arrays)).hexdigest()[:32]


def read_call(rs, q, back, dev_out=False):
    """phant_gpu_resident_state_read into fresh host arrays (dev_out: the account statuses on the device): rc, root, digest"""
    import torch

    n, m = q.n_accounts, q.n_slots
    r = [np.zeros(n, np.uint8), np.zeros(n, np.uint64), np.zeros((n, 32), np.uint8), np.zeros((n, 32), np.uint8),
         np.zeros((n, 32), np.uint8), np.zeros(m, np.uint8), np.zeros((m, 32), np.uint8)]
    ptrs = [gpu._ptr(a) if a.size else None for a in r]
    if dev_out:
        d = torch.zeros(n, dtype=torch.uint8, device="cuda")
        ptrs[0] = d.data_ptr()
    root = np.zeros(32, np.uint8)
    rc = rs.read_raw(q, back, gpu.StateReadValues(*ptrs), root)
    return rc, root.tobytes().hex(), digest(*r)


def range_call(rs, account_ranges, storage_ranges, back):
    """phant_gpu_resident_state_range into fresh host arrays sized by sum(max): rc, root, digest"""
    cat = lambda xs: np.frombuffer(b"".join(xs), np.uint8).copy() if xs else np.zeros(32, np.uint8)  # noqa: E731
    n, m = len(account_ranges), len(storage_ranges)
    ao, al = cat([r[0] for r in account_ranges]), cat([r[1] for r in account_ranges])
    amax = np.array([r[2] for r in account_ranges] or [0], np.uint32)
    sa, so, sl = (cat([r[i] for r in storage_ranges]) for i in range(3))
    smax = np.array([r[3] for r in storage_ranges] or [0], np.uint32)
    q = gpu.RangeRequest(n, gpu._ptr(ao), gpu._ptr(al), gpu._ptr(amax), m, gpu._ptr(sa), gpu._ptr(so), gpu._ptr(sl), gpu._ptr(smax))
    ea, es = max(int(amax[:n].sum()), 1), max(int(smax[:m].sum()), 1)
    r = [np.zeros(n + 1, np.uint64), np.zeros(max(n, 1), np.uint8), np.zeros((ea, 32), np.uint8), np.zeros(ea, np.uint64),
         np.zeros((ea, 32), np.uint8), np.zeros((ea, 32), np.uint8), np.zeros((ea, 32), np.uint8), np.zeros(m + 1, np.uint64),
         np.zeros(max(m, 1), np.uint8), np.zeros((es, 32), np.uint8), np.zeros((es, 32), np.uint8)]
    root = np.zeros(32, np.uint8)
    rc = rs.range_raw(q, back, gpu.RangeValues(*[gpu._ptr(a) for a in r]), root)
    return rc, root.tobytes().hex(), digest(*r)


def block_diff(rng, keys, n_new):
    d = Diff()
    for i, k in enumerate(keys):
        f = DELETE if i % 9 == 4 else (CLEAR if i % 11 == 5 else 0)
        d.accounts.append((k, f, i + 3, (i + 7).to_bytes(32, "big"), bytes(32)))
        if not f & DELETE:
            d.slots += [(i, rbytes(rng, 32), (j + 1).to_bytes(32, "big")) for j in range(i % 5)]
    for _ in range(n_new):
        d.accounts.append((rbytes(rng, 32), 0, 1, (1).to_bytes(32, "big"), bytes(32)))
        d.slots += [(len(d.accounts) - 1, rbytes(rng, 32), (9).to_bytes(32, "big"))]
    return d


def world_state_calls(ctx, rs, rng, keys, d):
    """codes, proofs, reads, ranges and a witness of a state with a journal of 3 applies (depth 4), then one refusal per rule"""
    import torch

    lib = gpu._lib()
    # codes: put (with a repeat and the empty code), a journaled block that names some of them, lookups, prune
    codes = [rbytes(rng, int(rng.integers(1, 3000))) for _ in range(40)]
    codes += [codes[3], b""]
    data, off = gpu._csr_bytes(codes)
    hashes = np.zeros((len(codes), 32), np.uint8)
    show(ctx, "state_put_codes", f"{rs.put_codes_raw(data, off, len(codes), hashes)} {digest(hashes)}")
    named = block_diff(rng, keys[900:1000], 10)
    named.accounts = [a[:4] + (hashes[i].tobytes(),) if i < 20 else a for i, a in enumerate(named.accounts)]
    show(ctx, "state_apply/journal/3", hexs(rs.apply(**named.arrays())))
    want = np.concatenate([hashes[:30], rng.integers(0, 256, (2, 32), dtype=np.uint8)])
    for tag, cap in (("small", 100), ("large", 1 << 20)):
        status, coff, buf = np.zeros(len(want), np.uint8), np.zeros(len(want) + 1, np.uint64), np.zeros(cap, np.uint8)
        rc = rs.codes_raw(want, len(want), status, coff, buf, cap)
        show(ctx, f"state_codes/{tag}", f"{rc} {digest(status, coff, buf)}")
    rc = lib.phant_gpu_resident_state_prune_codes(rs._h)
    info = rs.info()
    show(ctx, "state_prune_codes", f"{rc} {info['n_codes']} {info['code_bytes']}")

    # one request for prove and read: accounts of the last block and absent ones, slots of the last block
    acc = [a[0] for a in d.accounts[:60]] + [rbytes(rng, 32) for _ in range(5)]
    sl = [(ai, sk) for ai, sk, _ in d.slots if ai < 60][:80]
    q = rs._request(np.frombuffer(b"".join(acc), np.uint8), [ai for ai, _ in sl], np.frombuffer(b"".join(sk for _, sk in sl), np.uint8))
    rc, size = rs.prove_raw(q)
    show(ctx, "state_prove", f"{rc} {size.n_nodes} {size.nodes_bytes} {size.n_refs}")
    show(ctx, "state_prove_copy", " ".join(map(str, prove_copy(rs, q, size))))
    for back in (0, 2):
        show(ctx, f"state_read/{back}", " ".join(map(str, read_call(rs, q, back))))
    lo, hi = sorted([rbytes(rng, 32), rbytes(rng, 32)])
    ar = [(bytes(32), b"\xff" * 32, 40), (lo, hi, 500), (acc[7], acc[7], 1)]
    sr = [(d.accounts[ai][0], bytes(32), b"\xff" * 32, 3) for ai in sorted({ai for ai, _ in sl})[:6]]
    for back in (0, 2):
        show(ctx, f"state_range/{back}", " ".join(map(str, range_call(rs, ar, sr, back))))

    # a witness, then its copy (witness() makes both calls; here each prints its own return code)
    diff = rs._diff(**block_diff(rng, keys[1000:1100], 30).arrays())
    rc, wsize = rs.witness_raw(diff)
    show(ctx, "state_witness_raw", f"{rc} {wsize.n_nodes} {wsize.nodes_bytes}")
    show(ctx, "state_witness_copy", " ".join(map(str, witness_copy(rs, wsize))))

    # refusals: the device-pointer flag, a device-pointer output, `back` past the journal
    ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
    show(ctx, "refuse_flag/read", read_call(rs, q, 0)[0])
    show(ctx, "refuse_flag/put_codes", rs.put_codes_raw(data, off, len(codes), hashes))
    ctx.set_flags(0)
    show(ctx, "refuse_device_out/read", read_call(rs, q, 0, dev_out=True)[0])
    dstatus = torch.zeros(len(want), dtype=torch.uint8, device="cuda")
    show(ctx, "refuse_device_out/codes", rs.codes_raw(want, len(want), dstatus.data_ptr(), coff, None, 0))
    past = rs.info()["journal_applies"] + 1
    show(ctx, "refuse_back/read", read_call(rs, q, past)[0])
    show(ctx, "refuse_back/range", range_call(rs, ar, sr, past)[0])


def witness_copy(rs, size):
    """phant_gpu_resident_state_witness_copy into fresh host arrays sized by `size` (a WitnessSize): rc, digest"""
    nodes, noff = np.zeros(max(size.nodes_bytes, 1), np.uint8), np.zeros(size.n_nodes + 1, np.uint64)
    return rs.witness_copy_raw(nodes, noff), digest(nodes, noff)


def prove_copy(rs, q, size):
    """phant_gpu_resident_state_prove_copy of request q into fresh host arrays sized by `size` (a ProofSize): rc, digest"""
    n, m = q.n_accounts, q.n_slots
    pr = [np.zeros(max(size.nodes_bytes, 1), np.uint8), np.zeros(size.n_nodes + 1, np.uint64), np.zeros(max(size.n_refs, 1), np.uint64),
          np.zeros(n + m + 1, np.uint64), np.zeros((max(n + m, 1), 32), np.uint8), np.zeros(max(n + m, 1), np.uint8),
          np.zeros(max(n, 1), np.uint64), np.zeros((max(n, 1), 32), np.uint8), np.zeros((max(n, 1), 32), np.uint8),
          np.zeros((max(n, 1), 32), np.uint8), np.zeros((max(m, 1), 32), np.uint8)]
    return rs.prove_copy_raw(gpu.Proofs(*[gpu._ptr(a) for a in pr])), digest(*pr)


def trie_nodes_copy(rs, q, size):
    """phant_gpu_resident_state_trie_nodes_copy of request q into fresh host arrays sized by `size` (a WitnessSize): rc, digest"""
    n = q.n_paths
    r = [np.zeros(max(n, 1), np.uint8), np.zeros(n + 1, np.uint64), np.zeros(max(size.nodes_bytes, 1), np.uint8)]
    return rs.trie_nodes_copy_raw(gpu.TrieNodes(*[gpu._ptr(a) for a in r])), digest(*r)


def snap_copy(rs, q, size):
    """phant_gpu_resident_state_snap_ranges_copy of request q into fresh host arrays sized by `size` (a SnapSize): rc, digest"""
    n, m = q.n_account_requests, q.n_storage_requests
    z = lambda k, t=np.uint64: np.zeros(max(int(k), 1), t)  # noqa: E731
    r = [z(n + 1), z(32 * size.n_accounts, np.uint8), z(size.n_accounts + 1), z(size.account_bytes, np.uint8), z(m + 1),
         z(size.n_served + 1), z(32 * size.n_slots, np.uint8), z(size.n_slots + 1), z(size.slot_bytes, np.uint8), z(n + m + 1),
         z(size.n_refs), z(size.nodes_bytes, np.uint8), z(size.n_nodes + 1)]
    return rs.snap_ranges_copy_raw(gpu.SnapRanges(*[gpu._ptr(a) for a in r])), digest(*r)


def snap_request(rng, d):
    """account requests from 0 and from d's accounts at budgets 0 .. 2 MiB, one with its limit below its origin; storage
    requests over d's accounts with storage, with an absent account and an account d deletes among them, one from a slot key"""
    ff = b"\xff" * 32
    owners = [d.accounts[ai][0] for ai in sorted({ai for ai, _, _ in d.slots})[:6]]
    ar = [(bytes(32), ff, b) for b in (0, 37, 1000, 2 << 20)] + [(a[0], ff, int(b)) for a, b in zip(d.accounts[:8], rng.integers(0, 5000, 8))]
    ar.append((d.accounts[2][0], d.accounts[1][0], 100))
    s0 = next(sk for ai, sk, _ in d.slots)
    sr = [(owners[:3], bytes(32), ff, 100), (owners, bytes(32), ff, 1 << 20), (owners[2:] + [rbytes(rng, 32), d.accounts[4][0]], bytes(32), ff, 4000),
          ([d.accounts[d.slots[0][0]][0]], s0, ff, 50)]
    return gpu.ResidentState._snap_request(ar, sr)


def trie_node_request(rng, d):
    """account paths (the root, prefixes of d's accounts, a full 64-nibble key, one path twice) and storage paths (the root and
    prefixes of slot keys of some accounts with storage, the root and a prefix under an account d deletes and an absent one)"""
    owners = sorted({ai for ai, _, _ in d.slots})[:4]
    sa = [d.accounts[ai][0] for ai in owners] + [d.accounts[4][0], rbytes(rng, 32)]  # block_diff deletes account 4
    items = [(0, bytes(32), 0)] + [(0, a[0], int(rng.integers(1, 8))) for a in d.accounts[:12]] + [(0, d.accounts[1][0], 64)]
    items.append(items[3])
    for t, ai in enumerate(owners):
        items.append((1 + t, bytes(32), 0))
        items += [(1 + t, sk, int(rng.integers(1, 5))) for a, sk, _ in d.slots if a == ai][:3]
        items.append((1 + t, next(sk for a, sk, _ in d.slots if a == ai), 64))
    items += [(len(owners) + 1, bytes(32), 0), (len(owners) + 2, bytes(32), 0), (len(owners) + 2, rbytes(rng, 32), 3)]
    return rs_trie_node_request(items, sa)


def rs_trie_node_request(items, storage_accounts):
    """items: [(trie, 32-byte path, nibbles)]"""
    sa = np.frombuffer(b"".join(storage_accounts), np.uint8).copy() if storage_accounts else None
    paths = np.frombuffer(b"".join(p for _, p, _ in items), np.uint8).copy() if items else np.zeros(0, np.uint8)
    return gpu.ResidentState._trie_node_request(paths, [n for _, _, n in items], [t for t, _, _ in items], sa)


def node_set_calls(ctx, rs, rng, keys, d):
    """the four calls that hold a result until it is copied (witness, prove, trie_nodes, snap_ranges): trie_nodes and
    snap_ranges on mixed requests, each of their refusals and the refusals of the other two, empty requests, each copy with
    nothing held, each kind after each kind, and all four on a fork(1); d is the state's last block but one"""
    import torch

    tq = trie_node_request(rng, d)
    acc = [a[0] for a in d.accounts[:40]] + [rbytes(rng, 32) for _ in range(3)]
    sl = [(ai, sk) for ai, sk, _ in d.slots if ai < 40][:50]
    pq = rs._request(np.frombuffer(b"".join(acc), np.uint8), [ai for ai, _ in sl], np.frombuffer(b"".join(sk for _, sk in sl), np.uint8))
    wd = rs._diff(**block_diff(rng, keys[1100:1160], 10).arrays())
    sq = snap_request(rng, d)
    sizes = {}

    def size_call(name, q):
        rc, size = {"witness": rs.witness_raw, "prove": rs.prove_raw, "trie_nodes": rs.trie_nodes_raw, "snap_ranges": rs.snap_ranges_raw}[name](q)
        sizes[name] = size
        if name == "snap_ranges":
            return f"{rc} " + " ".join(str(getattr(size, f)) for f, _ in gpu.SnapSize._fields_[:8])
        return f"{rc} {size.n_nodes} {size.nodes_bytes}" + (f" {size.n_refs}" if name == "prove" else "")

    def copy_call(name, q):
        size = sizes.get(name) or (gpu.ProofSize() if name == "prove" else gpu.SnapSize() if name == "snap_ranges" else gpu.WitnessSize())
        rc, dg = (witness_copy(rs, size) if name == "witness" else prove_copy(rs, q, size) if name == "prove" else
                  snap_copy(rs, q, size) if name == "snap_ranges" else trie_nodes_copy(rs, q, size))
        return f"{rc} {dg}"

    req = {"witness": wd, "prove": pq, "trie_nodes": tq, "snap_ranges": sq}
    for name in req:
        show(ctx, f"held/copy_nothing/{name}", copy_call(name, req[name]))
    show(ctx, "trie_nodes", size_call("trie_nodes", tq))
    show(ctx, "trie_nodes_copy", copy_call("trie_nodes", tq))
    show(ctx, "snap_ranges", size_call("snap_ranges", sq))
    show(ctx, "snap_ranges_copy", copy_call("snap_ranges", sq))
    # each kind held, then each kind: the first one's copy finds nothing unless both are the same kind
    for a in req:
        for b in req:
            show(ctx, f"held/{a}/{b}/size", f"{size_call(a, req[a])} {size_call(b, req[b])}")
            show(ctx, f"held/{a}/{b}/copy", f"{copy_call(a, req[a])} {copy_call(b, req[b])} {rs.info()['device_bytes']}")

    # empty requests hold an empty result; trie nodes whose tries hold no key build no node set
    empty = {"witness": rs._diff(**Diff().arrays()), "prove": rs._request(np.zeros(0, np.uint8)), "trie_nodes": rs_trie_node_request([], []),
             "snap_ranges": rs._snap_request()}
    for name, q in empty.items():
        show(ctx, f"empty/{name}", f"{size_call(name, q)} {copy_call(name, q)}")
    no_key = rs_trie_node_request([(1, bytes(32), 0), (1, bytes(32), 2), (2, bytes(32), 0)], [rbytes(rng, 32), d.accounts[4][0]])
    show(ctx, "trie_nodes/no_key", f"{size_call('trie_nodes', no_key)} {copy_call('trie_nodes', no_key)}")

    # refusals: each ends with nothing held
    p2, l2, t2 = np.zeros(64, np.uint8), np.array([0, 3], np.uint8), np.array([0, 1], np.uint32)
    a1, a2 = (np.frombuffer(d.accounts[0][0] * r, np.uint8).copy() for r in (1, 2))
    l65, t_2 = np.array([0, 65], np.uint8), np.array([0, 2], np.uint32)
    dp = torch.zeros(64, dtype=torch.uint8, device="cuda")
    Q = gpu.TrieNodeRequest
    bad = {"null_paths": Q(2, None, l2.ctypes.data, None, 0, None), "null_lengths": Q(2, p2.ctypes.data, None, None, 0, None),
           "length_65": Q(2, p2.ctypes.data, l65.ctypes.data, None, 0, None),
           "trie_past_accounts": Q(2, p2.ctypes.data, l2.ctypes.data, t_2.ctypes.data, 1, a1.ctypes.data),
           "null_storage_accounts": Q(2, p2.ctypes.data, l2.ctypes.data, t2.ctypes.data, 1, None),
           "storage_account_twice": Q(2, p2.ctypes.data, l2.ctypes.data, t2.ctypes.data, 2, a2.ctypes.data),
           "too_many_paths": Q((1 << 28) + 1, p2.ctypes.data, l2.ctypes.data, None, 0, None),
           "device_paths": Q(2, dp.data_ptr(), l2.ctypes.data, None, 0, None)}
    for tag, q in bad.items():
        size_call("trie_nodes", tq)
        ctx.reset_stats()
        show(ctx, f"refuse_trie_nodes/{tag}", f"{size_call('trie_nodes', q)} {copy_call('trie_nodes', tq)}")
    show(ctx, "trie_nodes/null_unused_storage_accounts", size_call("trie_nodes", Q(2, p2.ctypes.data, l2.ctypes.data, None, 5, None)))
    S = gpu.SnapRequest
    o1, b1, f_bad, f_down = np.zeros(64, np.uint8), np.array([100, 100], np.uint64), np.array([1, 1], np.uint64), np.array([0, 2, 1], np.uint64)
    f_one = np.array([0, 1], np.uint64)
    sbad = {"null_origin": S(1, None, o1.ctypes.data, b1.ctypes.data, 0, None, None, None, None, None),
            "null_bytes": S(1, o1.ctypes.data, o1.ctypes.data, None, 0, None, None, None, None, None),
            "null_first": S(0, None, None, None, 1, None, o1.ctypes.data, o1.ctypes.data, o1.ctypes.data, b1.ctypes.data),
            "first_not_0": S(0, None, None, None, 1, f_bad.ctypes.data, o1.ctypes.data, o1.ctypes.data, o1.ctypes.data, b1.ctypes.data),
            "first_down": S(0, None, None, None, 2, f_down.ctypes.data, o1.ctypes.data, o1.ctypes.data, o1.ctypes.data, b1.ctypes.data),
            "null_accounts": S(0, None, None, None, 1, f_one.ctypes.data,
                               None, o1.ctypes.data, o1.ctypes.data, b1.ctypes.data),
            "too_many": S((1 << 28) + 1, o1.ctypes.data, o1.ctypes.data, b1.ctypes.data, 0, None, None, None, None, None),
            "device_origin": S(1, dp.data_ptr(), o1.ctypes.data, b1.ctypes.data, 0, None, None, None, None, None)}
    for tag, q in sbad.items():
        size_call("snap_ranges", sq)
        ctx.reset_stats()
        show(ctx, f"refuse_snap_ranges/{tag}", f"{size_call('snap_ranges', q)} {copy_call('snap_ranges', sq)}")
    ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
    show(ctx, "refuse_flag/trie_nodes", size_call("trie_nodes", tq))
    show(ctx, "refuse_flag/snap_ranges", size_call("snap_ranges", sq))
    ctx.set_flags(0)
    dup = Diff([d.accounts[0], d.accounts[1], d.accounts[0]])
    s0 = d.accounts[0][0]
    twice = {"witness/account_twice": ("witness", rs._diff(**dup.arrays())),
             "witness/slot_twice": ("witness", rs._diff(**Diff(d.accounts[:2], [(1, s0, s0), (0, s0, s0), (1, s0, s0)]).arrays())),
             "prove/account_twice": ("prove", rs._request(a2)),
             "prove/slot_twice": ("prove", rs._request(a1, [0, 0], np.frombuffer(s0 * 2, np.uint8)))}
    for tag, (name, q) in twice.items():
        size_call(name, req[name])
        ctx.reset_stats()
        show(ctx, f"refuse/{tag}", f"{size_call(name, q)} {copy_call(name, req[name])}")

    # all three at the root one apply back, on a fork
    f = rs.fork(1)
    show(ctx, "state_fork/1", hexs(f.root()))
    rs, sizes = f, {}  # size_call and copy_call now go to the fork
    for name in req:
        show(ctx, f"fork/{name}", f"{size_call(name, req[name])} {copy_call(name, req[name])}")
    f.close()


def rc_of(f):
    """f()'s return code: 0, or the code of the error it raised"""
    try:
        f()
        return 0
    except gpu.PhantGpuError as e:
        return e.code


def on_device(*arrays):
    """numpy arrays as device tensors, ready for the library's stream"""
    import torch

    signed = {np.dtype(np.uint32): np.int32, np.dtype(np.uint64): np.int64}  # same bytes, dtypes torch copies everywhere
    out = [torch.from_numpy(a.view(signed.get(a.dtype, a.dtype))).cuda() for a in arrays]
    torch.cuda.synchronize()
    return out


def witness_calls(ctx, data, off, keys, root):
    """W over a node set with host pointers, with device pointers, and with no node"""
    nk = len(keys) // 32
    outs = lambda: [np.zeros((nk + 63) // 64, np.uint64), np.zeros(nk, np.uint8), np.zeros(nk, np.uint64), np.zeros(nk, np.uint32)]  # noqa: E731
    for tag, nn in (("host", len(off) - 1), ("no_nodes", 0)):
        o = outs()
        rc = rc_of(lambda: ctx.verify_witness(nn, data if nn else None, off if nn else None, nk, keys, root, 1, *o))
        show(ctx, f"verify_witness/{tag}", f"{rc} {digest(*o)}")
    st = np.zeros(nk, np.uint8)
    rc = rc_of(lambda: ctx.verify_witness(len(off) - 1, data, off, nk, keys, root, 1, None, st))
    show(ctx, "verify_witness/host_status_only", f"{rc} {digest(st)}")
    rc = rc_of(lambda: ctx.verify_witness(len(off) - 1, data, off, nk, keys, np.tile(root, 2), 2, *outs()))
    show(ctx, "verify_witness/refused_n_roots", rc)
    o = outs()
    d_in, d_out = on_device(data, off, keys, root), on_device(*o)
    ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
    rc = rc_of(lambda: ctx.verify_witness(len(off) - 1, d_in[0], d_in[1], nk, d_in[2], d_in[3], 1, *d_out, nodes_bytes=int(off[-1])))
    ctx.synchronize()
    ctx.set_flags(0)
    show(ctx, "verify_witness/device", f"{rc} {digest(*[t.cpu().numpy() for t in d_out])}")


def read_state_calls(ctx, data, off, akeys, root, sacc, skeys, rng):
    """P over a node set with host pointers, with device pointers, and with no node; with codes, with each output left out,
    and refused"""
    na, ns = len(akeys) // 32, len(sacc)
    names = ("account_status", "nonce", "balance32", "storage_root32", "code_hash32", "code_index", "slot_status", "slot_vals32")
    outs = lambda: [np.zeros(na, np.uint8), np.zeros(na, np.uint64), np.zeros(32 * na, np.uint8), np.zeros(32 * na, np.uint8),  # noqa: E731
                    np.zeros(32 * na, np.uint8), np.zeros(na, np.uint32), np.zeros(ns, np.uint8), np.zeros(32 * ns, np.uint8)]
    for tag, nn in (("host", len(off) - 1), ("no_nodes", 0)):
        o = outs()
        rc = rc_of(lambda: ctx.read_state(nn, data if nn else None, off if nn else None, na, akeys, root, 1, ns, skeys, sacc,
                                          **dict(zip(names, o))))
        show(ctx, f"read_state/{tag}", f"{rc} {digest(*o)}")
    codes, coff = csr([rbytes(rng, int(rng.integers(0, 400))) for _ in range(7)], np.uint64)
    o = outs()
    rc = rc_of(lambda: ctx.read_state(len(off) - 1, data, off, na, akeys, root, 1, ns, skeys, sacc, n_codes=7, codes=codes, code_off=coff,
                                      **dict(zip(names, o))))
    show(ctx, "read_state/host_codes", f"{rc} {digest(*o)}")
    for i, name in enumerate(names):
        o = outs()
        kw = {k: (None if k == name else v) for k, v in zip(names, o)}
        rc = rc_of(lambda: ctx.read_state(len(off) - 1, data, off, na, akeys, root, 1, ns, skeys, sacc, n_codes=7, codes=codes, code_off=coff, **kw))
        show(ctx, f"read_state/host_without_{name}", f"{rc} {digest(*[a for j, a in enumerate(o) if j != i])}")
    bad = sacc.copy()
    bad[-1] = na
    rc = rc_of(lambda: ctx.read_state(len(off) - 1, data, off, na, akeys, root, 1, ns, skeys, bad, **dict(zip(names, outs()))))
    show(ctx, "read_state/refused_slot_account", rc)
    for tag, n_codes in (("device", 0), ("device_codes", 7)):
        o = outs()
        d_in, d_out = on_device(data, off, akeys, root, skeys, sacc, padded(codes), coff), on_device(*o)
        ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
        rc = rc_of(lambda: ctx.read_state(len(off) - 1, d_in[0], d_in[1], na, d_in[2], d_in[3], 1, ns, d_in[4], d_in[5], n_codes=n_codes,
                                          codes=d_in[6] if n_codes else None, code_off=d_in[7] if n_codes else None,
                                          nodes_bytes=int(off[-1]), codes_bytes=int(coff[-1]) if n_codes else 0, **dict(zip(names, d_out))))
        ctx.synchronize()
        ctx.set_flags(0)
        show(ctx, f"read_state/{tag}", f"{rc} {digest(*[t.cpu().numpy() for t in d_out])}")


def padded(data):
    """a device input with the 64 readable bytes of tail the Keccak kernels may touch"""
    return np.concatenate([data, np.zeros(64, np.uint8)])


def device_call(ctx, f):
    """f()'s return code with device pointers, once the context's stream is done"""
    ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
    try:
        rc = rc_of(f)
        ctx.synchronize()
    finally:
        ctx.set_flags(0)
    return rc


def host_of(*tensors):
    return [t.cpu().numpy() for t in tensors]


def keccak_calls(ctx, rng):
    """K with host pointers, with device pointers, in its asynchronous form, and refused"""
    data, off = csr([rbytes(rng, int(rng.integers(0, 300))) for _ in range(6000)], np.uint64)
    n = len(off) - 1
    out = np.zeros((n, 32), np.uint8)
    rc = rc_of(lambda: ctx.keccak256_batch(data, off, n, out))
    show(ctx, "keccak256_batch/host", f"{rc} {digest(out)}")
    d_data, d_off, d_out, d_out2 = on_device(padded(data), off, out, out)
    rc = device_call(ctx, lambda: ctx.keccak256_batch(d_data, d_off, n, d_out))
    show(ctx, "keccak256_batch/device", f"{rc} {digest(*host_of(d_out))}")
    rc = device_call(ctx, lambda: ctx.keccak256_batch_async(d_data, d_off, n, int(off[-1]), d_out2))
    show(ctx, "keccak256_batch_async/device", f"{rc} {digest(*host_of(d_out2))}")
    rc = rc_of(lambda: ctx.keccak256_batch_async(d_data, d_off, n, int(off[-1]), d_out2))
    show(ctx, "keccak256_batch_async/refused_host_flags", rc)
    rc = rc_of(lambda: ctx.keccak256_batch(data, None, n, out))
    show(ctx, "keccak256_batch/refused_no_offsets", rc)


def verify_proofs_calls(ctx, oracle):
    """V in chain form (the chunked host pipeline, fused and unfused, and each output left out) and in deduplicated form, with
    host and device pointers, sharded at world 1, the block reject counts of its verdicts, and refused"""
    n = 10000  # at PHANT_GPU_CHUNK_MB=1 the chain form crosses in three chunks
    nodes, noff, first, keys, roots = oracle.synth_c2(n, depth=8, first=5)
    words = (n + 63) // 64
    outs = lambda: [np.zeros(words, np.uint64), np.zeros(n, np.uint8), np.zeros(n, np.uint64), np.zeros(n, np.uint32)]  # noqa: E731
    for tag, flags in (("fused", 0), ("unfused", gpu.FLAG_UNFUSED_WALK)):
        o = outs()
        ctx.set_flags(flags)
        rc = rc_of(lambda: ctx.verify_proofs(n, nodes, noff, first, keys, roots, n, *o))
        ctx.set_flags(0)
        show(ctx, f"verify_proofs/chain_host_{tag}", f"{rc} {digest(*o)}")
    for i in range(4):
        o = outs()
        kept = [None if j != i else a for j, a in enumerate(o)]
        rc = rc_of(lambda: ctx.verify_proofs(n, nodes, noff, first, keys, roots, n, *kept))
        show(ctx, f"verify_proofs/chain_host_only_{i}", f"{rc} {digest(o[i])}")
    rc = rc_of(lambda: ctx.verify_proofs(n, nodes, noff, first, keys, roots, 2, *outs()))
    show(ctx, "verify_proofs/refused_n_roots", rc)
    d_in, d_out = on_device(padded(nodes), noff, first, keys, roots), on_device(*outs())
    rc = device_call(ctx, lambda: ctx.verify_proofs(n, *d_in, n, *d_out))
    show(ctx, "verify_proofs/chain_device", f"{rc} {digest(*host_of(*d_out))}")

    # deduplicated form: the first 1,000 proofs twice over one copy of their nodes, chains as index lists
    h, hn = 1000, int(first[1000])
    m = 2 * h
    dnodes, doff = nodes[:int(noff[hn])].copy(), noff[:hn + 1].copy()
    refs = np.tile(np.arange(hn, dtype=np.uint64), 2)
    dfirst = np.concatenate([first[:h + 1], first[1:h + 1] + np.uint64(hn)])
    dkeys, droots = np.tile(keys[:32 * h], 2), np.tile(roots[:32 * h], 2)
    mo = lambda: [np.zeros((m + 63) // 64, np.uint64), np.zeros(m, np.uint8), np.zeros(m, np.uint64), np.zeros(m, np.uint32)]  # noqa: E731
    o = mo()
    rc = rc_of(lambda: ctx.verify_proofs(m, dnodes, doff, dfirst, dkeys, droots, m, *o, n_nodes=hn, node_index=refs))
    show(ctx, "verify_proofs/dedup_host", f"{rc} {digest(*o)}")
    o = mo()
    rc = rc_of(lambda: ctx.verify_proofs(m, dnodes, doff, dfirst, dkeys, droots, m, None, o[1], n_nodes=hn, node_index=refs))
    show(ctx, "verify_proofs/dedup_host_status_only", f"{rc} {digest(o[1])}")
    bad = refs.copy()
    bad[-1] = hn
    rc = rc_of(lambda: ctx.verify_proofs(m, dnodes, doff, dfirst, dkeys, droots, m, *mo(), n_nodes=hn, node_index=bad))
    show(ctx, "verify_proofs/dedup_refused_index", rc)
    dd_in, dd_out = on_device(padded(dnodes), doff, dfirst, dkeys, droots, refs), on_device(*mo())
    rc = device_call(ctx, lambda: ctx.verify_proofs(m, *dd_in[:5], m, *dd_out, n_nodes=hn, nodes_bytes=int(doff[-1]),
                                                    node_index=dd_in[5]))
    show(ctx, "verify_proofs/dedup_device", f"{rc} {digest(*host_of(*dd_out))}")

    # sharded at world 1: host pointers read the bitmap the plain call left on the device
    gb, st = np.zeros(gpu.sharded_bitmap_words(n, 1), np.uint64), np.zeros(n, np.uint8)
    rc = rc_of(lambda: ctx.verify_proofs_sharded(n, n, nodes, noff, first, keys, roots, n, gb, st))
    show(ctx, "verify_proofs_sharded/host", f"{rc} {digest(gb, st)}")
    gb2 = np.zeros(gpu.sharded_bitmap_words(m, 1), np.uint64)
    rc = rc_of(lambda: ctx.verify_proofs_sharded(m, m, dnodes, doff, dfirst, dkeys, droots, m, gb2, None, n_nodes=hn, node_index=refs))
    show(ctx, "verify_proofs_sharded/dedup_host", f"{rc} {digest(gb2)}")
    d_gb, d_st = on_device(gb, st)
    rc = device_call(ctx, lambda: ctx.verify_proofs_sharded(n, n, *d_in, n, d_gb, d_st))
    show(ctx, "verify_proofs_sharded/device", f"{rc} {digest(*host_of(d_gb, d_st))}")
    rc = rc_of(lambda: ctx.verify_proofs_sharded(n - 1, n, nodes, noff, first, keys, roots, n, gb, st))
    show(ctx, "verify_proofs_sharded/refused_shard", rc)

    # block reject counts over the chain form's status bytes
    block = (np.arange(n) * 37 // n).astype(np.uint32)
    counts = np.zeros(37, np.uint32)
    rc = rc_of(lambda: ctx.block_reject_counts(st, block, n, 37, counts))
    show(ctx, "block_reject_counts/host", f"{rc} {digest(counts)}")
    rc = rc_of(lambda: ctx.block_reject_counts(None, None, 0, 37, counts))
    show(ctx, "block_reject_counts/host_no_proofs", f"{rc} {digest(counts)}")
    d_st, d_block, d_counts = on_device(st, block, counts)
    rc = device_call(ctx, lambda: ctx.block_reject_counts(d_st, d_block, n, 37, d_counts))
    show(ctx, "block_reject_counts/device", f"{rc} {digest(*host_of(d_counts))}")
    rc = rc_of(lambda: ctx.block_reject_counts(st, block, n, 0, counts))
    show(ctx, "block_reject_counts/refused_no_blocks", rc)


def bloom_calls(ctx, rng):
    """B with host pointers, with device pointers, with no item, and refused"""
    n, nb = 3000, 50
    items, ioff = csr([rbytes(rng, int(rng.integers(0, 80))) for _ in range(n)], np.uint64)
    owner = rng.integers(0, nb, n).astype(np.uint32)
    blooms = np.zeros((nb, 256), np.uint8)
    rc = rc_of(lambda: ctx.logs_bloom(items, ioff, owner, n, nb, blooms))
    show(ctx, "logs_bloom/host", f"{rc} {digest(blooms)}")
    empty = np.ones((nb, 256), np.uint8)
    rc = rc_of(lambda: ctx.logs_bloom(None, None, None, 0, nb, empty))
    show(ctx, "logs_bloom/host_no_items", f"{rc} {digest(empty)}")
    d_items, d_ioff, d_owner, d_blooms = on_device(padded(items), ioff, owner, blooms)
    rc = device_call(ctx, lambda: ctx.logs_bloom(d_items, d_ioff, d_owner, n, nb, d_blooms))
    show(ctx, "logs_bloom/device", f"{rc} {digest(*host_of(d_blooms))}")
    bad = owner.copy()
    bad[-1] = nb
    rc = rc_of(lambda: ctx.logs_bloom(items, ioff, bad, n, nb, blooms))
    show(ctx, "logs_bloom/refused_owner", rc)


def ecrecover_calls(ctx, rng):
    """sender recovery with and without public keys and addresses, with device pointers, and refused"""
    n = 2000
    hashes = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    sigs = rng.integers(0, 256, (n, 65), dtype=np.uint8)
    sigs[:, 64] = rng.integers(0, 5, n)  # recovery ids 0..3 and some invalid ones
    for tag, want_pub, want_addr in (("all", True, True), ("no_pubkeys", False, True), ("no_addresses", True, False), ("ok_only", False, False)):
        pub, addr, ok = np.zeros((n, 65), np.uint8), np.zeros((n, 20), np.uint8), np.full(n, 7, np.uint8)
        rc = rc_of(lambda: ctx.ecrecover_batch(hashes, sigs, n, pub if want_pub else None, addr if want_addr else None, ok))
        show(ctx, f"ecrecover_batch/host_{tag}", f"{rc} {digest(pub, addr, ok)}")
    d_h, d_s, d_pub, d_addr, d_ok = on_device(hashes, sigs, np.zeros((n, 65), np.uint8), np.zeros((n, 20), np.uint8), np.zeros(n, np.uint8))
    rc = device_call(ctx, lambda: ctx.ecrecover_batch(d_h, d_s, n, d_pub, d_addr, d_ok))
    show(ctx, "ecrecover_batch/device", f"{rc} {digest(*host_of(d_pub, d_addr, d_ok))}")
    rc = rc_of(lambda: ctx.ecrecover_batch(hashes, sigs, n, None, None, None))
    show(ctx, "ecrecover_batch/refused_no_ok", rc)


def range_calls(ctx, oracle, rng):
    """G: one batch of honest answers (some with more), a WHOLE range, an empty answer past the last key, an empty-root
    range and an answer with one entry's value changed"""
    t = random_tries(oracle)[0]
    cases = [(t.root, o, e, n, w) for o, e, n, w, _ in accept_cases(t, counts=(2,), limit=4, rng=rng)]
    cases.append((EMPTY_ROOT, bytes(32), [], [], False))
    cases += [c[1:] for c in mutations(t, t.keys[1], 4, rng) if c[0] == "value-byte"]
    nodes = list(dict.fromkeys(n for c in cases for n in c[3]))
    got = []
    rc = rc_of(lambda: got.extend(host.verify_ranges(ctx, [(r, o, e, w) for r, o, e, _, w in cases], nodes)))
    show(ctx, "verify_ranges", f"{rc} {got}")


def main():
    import torch

    rng = np.random.default_rng(20261016)
    oracle = oracle_lib.get()
    ctx = gpu.Context(0)
    ctx.reset_stats()

    # M: one trie with 32-byte keys (slot layout), one with short keys that are prefixes of each other (general layout)
    k, ko, v, vo, n = mpt_inputs(rng, 3000, 32)
    show(ctx, "mpt_root/32", hexs(ctx.mpt_root(k, ko, v, vo, n)))
    k, ko, v, vo, n = mpt_inputs(rng, 3000, 3)
    show(ctx, "mpt_root/short", hexs(ctx.mpt_root(k, ko, v, vo, n)))
    segs, parts = [0], []
    for t in range(40):
        parts.append(mpt_inputs(rng, int(rng.integers(0, 200)), 8 if t % 2 else 32))
        segs.append(segs[-1] + parts[-1][4])
    keys = [bytes(p[0][p[1][i]:p[1][i + 1]]) for p in parts for i in range(p[4])]
    vals = [bytes(p[2][p[3][i]:p[3][i + 1]]) for p in parts for i in range(p[4])]
    k, ko = csr(keys, np.uint32)
    v, vo = csr(vals, np.uint64)
    show(ctx, "mpt_roots", hexs(ctx.mpt_roots(k, ko, v, vo, np.array(segs, np.uint32), len(parts))))
    # more than 8,192 keys of 32 bytes: the slot layout with one BFS launch per level (its own generator, as below)
    xrng = np.random.default_rng(20261020)
    big_keys = sorted({rbytes(xrng, 32) for _ in range(12000)})
    k, ko = csr(big_keys, np.uint32)
    v, vo = csr([rbytes(xrng, int(xrng.integers(1, 120))) for _ in big_keys], np.uint64)
    show(ctx, "mpt_root/32_level_bfs", hexs(ctx.mpt_root(k, ko, v, vo, len(big_keys))))

    # S
    a = accounts(rng, 5000)
    show(ctx, "state_root", hexs(ctx.state_root(*a)))
    out, mask = ctx.state_subtree_roots(*accounts(rng, 3000))
    show(ctx, "state_subtree_roots", f"{hexs(out)} {mask:#x}")

    # U kind 0: host pointers (fused frontier path), device pointers and an oversized value (general path)
    t0 = ctx.trie_open(5, kind=0)
    show(ctx, "trie0_open", hexs(t0.root()))
    kk = rng.integers(0, 256, (4000, 32), dtype=np.uint8)
    pos = rng.choice(16 ** 5, 4000, replace=False) << 4  # distinct leaf positions: the first 5 nibbles
    kk[:, 0], kk[:, 1], kk[:, 2] = pos >> 16, (pos >> 8) & 255, (pos & 255) | (kk[:, 2] & 15)
    vv, voff = csr([rbytes(rng, int(rng.integers(1, 200))) for _ in range(4000)], np.uint32)
    show(ctx, "trie0_update/host", hexs(t0.update(kk, vv, voff, 4000)))
    dk, dv, dvo = (torch.from_numpy(x).cuda() for x in (kk[:1000].copy(), vv, voff[:1001].copy()))
    torch.cuda.synchronize()
    ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
    r = t0.update(dk, dv, dvo, 1000)
    ctx.set_flags(0)
    show(ctx, "trie0_update/device", hexs(r))
    big, boff = csr([rbytes(rng, 600 if i % 3 == 0 else 40) for i in range(500)], np.uint32)
    show(ctx, "trie0_update/big", hexs(t0.update(kk[1000:1500].copy(), big, boff, 500)))
    # refused: two keys on one leaf position, on the fused and on the general leaf path; the root stays
    clash = kk[2000:2050].copy()
    clash[49] = clash[0]
    clash[49, 31] ^= 1
    for tag, sizes in (("fused", [40] * 50), ("general", [600] + [40] * 49)):
        cv, coff = csr([rbytes(xrng, z) for z in sizes], np.uint32)
        show(ctx, f"trie0_update/refused_{tag}", f"{rc_of(lambda: t0.update(clash, cv, coff, 50))} {hexs(t0.root())}")
    t0.close()

    # U kind 1: inserts that deepen the dense top, then deletes and changes
    t1 = ctx.trie_open(0, kind=1)
    live = []
    for step, n_ins in enumerate((200, 6000, 60000)):
        ins = rng.integers(0, 256, (n_ins, 32), dtype=np.uint8)
        vals, off = csr([rbytes(rng, int(rng.integers(1, 90))) for _ in range(n_ins)], np.uint32)
        show(ctx, f"trie1_insert/{step}", hexs(t1.update(ins, vals, off, n_ins)))
        live += [bytes(x) for x in ins]
    ch = [live[i] for i in range(0, len(live), 7)]
    vals = [b"" if i % 2 else rbytes(rng, 50) for i in range(len(ch))]  # empty value: delete
    v, off = csr(vals, np.uint32)
    show(ctx, "trie1_delete_change", hexs(t1.update(np.frombuffer(b"".join(ch), np.uint8).copy(), v, off, len(ch))))
    # a key twice (refused; the root stays), then deletes down to under 3,000 keys, which lower the dense depth
    twice = np.frombuffer(b"".join(live[:20] + [live[3]]), np.uint8).copy()
    v, off = csr([rbytes(xrng, 30) for _ in range(21)], np.uint32)
    show(ctx, "trie1_update/key_twice", f"{rc_of(lambda: t1.update(twice, v, off, 21))} {hexs(t1.root())}")
    gone = live[3000:]
    v, off = csr([b""] * len(gone), np.uint32)
    show(ctx, "trie1_delete/lower_depth", hexs(t1.update(np.frombuffer(b"".join(gone), np.uint8).copy(), v, off, len(gone))))
    t1.close()

    # world state: apply, the witness of a block (node count and digest of the copied CSR), then apply with a journal and revert
    rs = ctx.resident_state()
    d0 = block_diff(rng, [], 4000)
    show(ctx, "state_apply/0", hexs(rs.apply(**d0.arrays())))
    keys = [a[0] for a in d0.accounts]
    nodes, off = rs.witness(**block_diff(rng, keys[:300], 200).arrays())
    show(ctx, "state_witness", f"{len(off) - 1} {hashlib.sha256(nodes.tobytes() + off.tobytes()).hexdigest()}")
    rs.set_journal(4)
    roots = []
    for b in range(3):
        d = block_diff(rng, keys[b * 300:(b + 1) * 300], 200)
        r, sr = rs.apply(**d.arrays(), storage_roots=True)
        roots.append(r)
        show(ctx, f"state_apply/journal/{b}", hexs([r, sr]))
    world_state_calls(ctx, rs, rng, keys, d)
    node_set_calls(ctx, rs, np.random.default_rng(20261018), keys, d)  # its own generator: the calls after it see what they saw before
    show(ctx, "state_revert/1", hexs(rs.revert(1)))
    show(ctx, "state_revert/2", hexs(rs.revert(2)))
    rs.close()

    # T: two blocks over one node set
    blocks = []
    for _ in range(2):
        m, d = random_case(oracle, rng, n_acc=300, n_slots=60)
        blocks.append((witness(oracle, m, d), m.root(), d))
    nodes = list(dict.fromkeys(n for b in blocks for n in b[0]))
    data, off = oracle_lib.csr(nodes, np.uint64)
    d = Diff()
    ablock = []
    for bi, (_, _, bd) in enumerate(blocks):
        base = len(d.accounts)
        d.accounts += bd.accounts
        d.slots += [(base + ai, sk, val) for ai, sk, val in bd.slots]
        ablock += [bi] * len(bd.accounts)
    pre = np.frombuffer(b"".join(b[1] for b in blocks), np.uint8)
    roots, status, sroots = ctx.transition_roots(data, off, pre, **d.arrays(), account_block=np.array(ablock, np.uint32), storage_roots=True)
    show(ctx, "transition_roots", f"{hexs([roots, sroots])} {list(status)}")
    # T's refusals: a key listed twice in one segment; a block whose witness lacks a node (status 3, not an error)
    dup = Diff()
    dup.accounts, dup.slots = d.accounts + [d.accounts[0]], list(d.slots)
    rc = rc_of(lambda: ctx.transition_roots(data, off, pre, **dup.arrays(), account_block=np.array(ablock + [ablock[0]], np.uint32)))
    show(ctx, "transition_roots/duplicate_key", rc)
    b0 = blocks[0][0]
    lost = next(x for x in b0[len(b0) // 2:] if x not in blocks[1][0])
    ldata, loff = oracle_lib.csr([x for x in nodes if x != lost], np.uint64)
    got = []
    rc = rc_of(lambda: got.append(ctx.transition_roots(ldata, loff, pre, **d.arrays(), account_block=np.array(ablock, np.uint32))))
    show(ctx, "transition_roots/missing_node", f"{rc} {hexs(got[0][0]) if got else ''} {got[0][1].tolist() if got else ''}")

    # W and P over block 0's node set: its accounts and some absent ones at its pre-state root, and its slots
    bd = blocks[0][2]
    akeys = np.frombuffer(b"".join([a[0] for a in bd.accounts] + [rbytes(rng, 32) for _ in range(4)]), np.uint8).copy()
    root = np.frombuffer(blocks[0][1], np.uint8).copy()
    bdata, boff = oracle_lib.csr(blocks[0][0], np.uint64)
    witness_calls(ctx, bdata, boff, akeys, root)
    sacc = np.array([ai for ai, _, _ in bd.slots], np.uint32)
    skeys = np.frombuffer(b"".join(sk for _, sk, _ in bd.slots), np.uint8).copy()
    read_state_calls(ctx, bdata, boff, akeys, root, sacc, skeys, np.random.default_rng(20261019))

    # G
    range_calls(ctx, oracle, rng)

    # K, V, B, sender recovery and block reject counts: their own generator, so the calls above see what they saw before
    srng = np.random.default_rng(20261019)
    keccak_calls(ctx, srng)
    verify_proofs_calls(ctx, oracle)
    bloom_calls(ctx, srng)
    ecrecover_calls(ctx, srng)
    ctx.close()


if __name__ == "__main__":
    main()
