"""Trie nodes by path (snap's GetTrieNodes) from the resident world state (phant_gpu_resident_state_trie_nodes + _copy).

The state is that of tools/resident_state_bench.py: 1,000,000 accounts and about 10M slots.  Two request shapes:

  heal    what a healing peer asks for in one call: 1,024 paths, account-trie paths at depths 0..8 and storage paths under
          64 accounts, drawn from nodes that exist, plus 10% paths with no node
  single  one existing account-trie path per call, many calls

Paths "that exist" are found by an untimed discovery call over prefixes of random keys.  Host wall clock around each
synchronous call (trie_nodes and the copy of its result to the host).  Every served node is checked without the CPU trie:
its keccak (through K) is the state root or its account's storage root (read from the state) for the empty path, and is
otherwise held as a 32-byte reference by the node served at the longest shorter prefix of its path, fetched in one untimed
call.  Reported: median and p99 ms per call, with launches, H2D / D2H bytes and Keccak messages of a call, and the card's
name and power limit read in the same run.

    python tools/resident_state_trie_nodes_bench.py [--accounts 1000000] [--scale 1.0] [--calls 200] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
from phant_b200 import gpu  # noqa: E402
from resident_state_bench import build_state, card  # noqa: E402


def packed(key, d):
    """the first d nibbles of a 32-byte key, zero padded"""
    b = bytearray(key[:(d + 1) // 2])
    if d & 1:
        b[-1] &= 0xf0
    return bytes(b).ljust(32, b"\x00")


class Request:
    def __init__(self, items, owners):
        """items: [(trie: 0 or 1 + index into owners, packed path, nibbles)]"""
        self.items, self.owners = items, owners
        self.paths = np.frombuffer(b"".join(p for _, p, _ in items), np.uint8).copy()
        self.lens = np.array([n for _, _, n in items], np.uint8)
        self.tries = np.array([t for t, _, _ in items], np.uint32)
        self.sa = np.ascontiguousarray(owners.reshape(-1)) if len(owners) else None

    def ask(self, st):
        return st.trie_nodes(self.paths, self.lens, self.tries, self.sa)


def check(ctx, st, req, status, blobs, root, sroots):
    """every served node hashes to its parent's reference (or to its trie's root): see the module docstring"""
    served = [i for i in range(len(status)) if status[i] == 1]
    if not served:
        return 0
    msgs = b"".join(blobs[i] for i in served)
    off = np.zeros(len(served) + 1, np.uint64)
    off[1:] = np.cumsum([len(blobs[i]) for i in served])
    dig = np.zeros((len(served), 32), np.uint8)
    ctx.keccak256_batch(np.frombuffer(msgs + bytes(16), np.uint8).copy(), off, len(served), dig)
    prefixes = [(t, packed(p, d), d) for i in served for t, p, n in [req.items[i]] for d in range(n)]
    ps, pb = Request(prefixes, req.owners).ask(st) if prefixes else ([], [])
    k = 0
    for j, i in enumerate(served):
        t, _, n = req.items[i]
        h = dig[j].tobytes()
        parent = None
        for d in range(n):
            if ps[k + d] == 1:
                parent = pb[k + d]
        k += n
        if n == 0:
            assert h == (root if t == 0 else sroots[t - 1])
        else:
            assert parent is not None and b"\xa0" + h in parent
    return len(served)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every storage size (0.01 for a quick run)")
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--heals", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    rng = np.random.default_rng(args.seed)
    gpu_name = card()
    na = args.accounts
    akeys, nonce, bal, code, slot_acc, skeys, svals, store = build_state(rng, na, args.scale)
    ctx = gpu.Context(0)
    st = ctx.resident_state()
    root = st.apply(akeys, nonce, bal, code, None, slot_acc, skeys, svals)
    del slot_acc, skeys, svals
    rich = np.array([a for a in sorted(store) if len(store[a].k) >= 2], np.int64)

    def discover(n_acc, n_st):
        """a heal-shaped request: existing account paths at depths 0..8, existing storage paths under 64 accounts, and 10%
        paths with no node (inside leaves and under absent accounts)"""
        owner_idx = rich[rng.choice(len(rich), 64, replace=False)]
        owners = np.ascontiguousarray(akeys[owner_idx])
        cand = [(0, packed(akeys[int(a)].tobytes(), int(d)), int(d)) for a, d in zip(rng.integers(0, na, 4 * n_acc), rng.integers(0, 9, 4 * n_acc))]
        for j, a in enumerate(owner_idx):
            ks = store[int(a)].k
            for x, d in zip(rng.integers(0, len(ks), 8 * n_st // 64), rng.integers(0, 9, 8 * n_st // 64)):
                cand.append((1 + j, packed(ks[int(x)].tobytes(), int(d)), int(d)))
        s, _ = Request(cand, owners).ask(st)
        acc = [c for c, x in zip(cand, s) if x == 1 and c[0] == 0]
        sto = [c for c, x in zip(cand, s) if x == 1 and c[0] > 0]
        items = [acc[int(i)] for i in rng.integers(0, len(acc), n_acc)] + [sto[int(i)] for i in rng.integers(0, len(sto), n_st)]
        none = [(0, akeys[int(a)].tobytes(), 63) for a in rng.integers(0, na, (n_acc + n_st) // 9)]
        items += none
        rng.shuffle(items)
        sr, _ = st.read(owners)
        return Request(items, owners), [sr["storage_root32"][j].tobytes() for j in range(64)]

    def timed(f):
        ctx.synchronize()
        ctx.reset_stats()
        t0 = time.perf_counter()
        out = f()
        return out, (time.perf_counter() - t0) * 1e3, ctx.stats()

    def row(ms, s, status, blobs):
        return dict(ms=ms, launches=s["launches"], h2d_bytes=s["h2d_bytes"], d2h_bytes=s["d2h_bytes"], keccak_msgs=s["keccak_msgs"],
                    served=int((status == 1).sum()), served_bytes=sum(len(b) for b in blobs))

    heal_rows, checked = [], 0
    for c in range(args.warmup + args.heals):
        req, sroots = discover(614, 307)
        (status, blobs), ms, s = timed(lambda: req.ask(st))
        checked += check(ctx, st, req, status, blobs, root, sroots)
        if c >= args.warmup:
            heal_rows.append(row(ms, s, status, blobs))
    single_rows = []
    pool, _ = discover(256, 64)
    pool = [it for it in pool.items if it[0] == 0 and it[2] < 63]
    for c in range(args.warmup + args.calls):
        req = Request([pool[c % len(pool)]], np.zeros((0, 32), np.uint8))
        (status, blobs), ms, s = timed(lambda: req.ask(st))
        checked += check(ctx, st, req, status, blobs, root, [])
        assert status[0] == 1
        if c >= args.warmup:
            single_rows.append(row(ms, s, status, blobs))

    def summary(rows):
        med = {k: round(float(np.median([x[k] for x in rows])), 3) for k in rows[0]}
        med["p99_ms"] = round(float(np.percentile([x["ms"] for x in rows], 99)), 3)
        return {"calls": len(rows), "median": med}

    print(json.dumps({"gpu": gpu_name, "accounts": na, "scale": args.scale, "heal": summary(heal_rows), "single": summary(single_rows),
                      "all_served_nodes_checked": True, "served_nodes_checked": checked}))
    st.close()


if __name__ == "__main__":
    main()
