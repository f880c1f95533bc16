#!/usr/bin/env python3
"""Call each trie builder entry point once on seeded inputs and print every result followed by the context's counters.
Run it against two builds of libphantgpu.so and diff the outputs: a host-side change (how scratch areas are sized and laid
out, say) must leave every result, launch count, copy size and Keccak message count as it was.
  python tools/trie_calls.py [path/to/libphantgpu.so] > trie_calls_<tag>.txt
Needs a GPU.
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from phant_b200 import gpu  # noqa: E402

if len(sys.argv) > 1:
    gpu.LIB_PATH = os.path.abspath(sys.argv[1])

import oracle_lib  # noqa: E402
from resident_state_model import CLEAR, DELETE, Diff  # noqa: E402
from test_transition_model import random_case  # noqa: E402
from transition_oracle import witness  # noqa: E402

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
    ctx.close()


if __name__ == "__main__":
    main()
