"""Range proofs checked on the GPU (phant_gpu_verify_ranges) against answers the resident world state serves.

The state is tools/resident_state_bench.py's: 1,000,000 accounts and about 10M slots.  Answers are served with
phant_gpu_resident_state_range plus _prove (the boundary proofs of each range's origin and last key), then checked with one
verify call per batch; every status must be 1 and every `more` must equal the range call's.  Shapes:

  snap    one call holding 64 account ranges of 5,000 entries with their boundary proofs, and one call holding a
          GetStorageRanges answer: 100 storage ranges of up to 1,000 slots from random accounts, every complete one WHOLE,
          the others proven from their origin
  full    the whole state verified in calls of at most --chunk entries: the accounts range by range, then every account's
          slots, many accounts per call (a full sync's checks); reported as entries/s

Times are host wall clock around the synchronous verify calls only (serving and encoding the answers are not timed).
Launches, H2D bytes and Keccak messages come from phant_gpu_stats.  Prints one JSON line with the card's name and power limit
read in the same run.

    python tools/range_proof_bench.py [--accounts 1000000] [--scale 1.0] [--calls 10] [--chunk 1048576]
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

ZERO, ALL = bytes(32), b"\xff" * 32


def rlp_trimmed(rows):
    """rlp of each row with its leading zero bytes dropped (an integer, a slot value) -> (n x (w + 1) matrix, first column)"""
    n, w = rows.shape
    nz = rows != 0
    z = np.where(nz.any(axis=1), nz.argmax(axis=1), w)
    ln = w - z
    r = np.arange(n)
    single = (ln == 1) & (rows[r, np.minimum(z, w - 1)] < 0x80)
    m = np.zeros((n, w + 1), np.uint8)
    m[:, 1:] = rows
    start = np.where(ln == 0, w, np.where(single, z + 1, z))
    m[r, start] = np.where(ln == 0, 0x80, np.where(single, m[r, start], 0x80 + ln))
    return m, start


def pack(parts):
    """[(matrix, first column)] of n rows each -> the rows' concatenated tails as CSR (uint8 data, uint64 offsets)"""
    m = np.concatenate([p for p, _ in parts], axis=1)
    mask = [np.arange(p.shape[1])[None, :] >= s[:, None] for p, s in parts]
    mask = np.concatenate(mask, axis=1)
    off = np.zeros(len(m) + 1, np.uint64)
    off[1:] = np.cumsum(mask.sum(axis=1))
    return np.ascontiguousarray(m[mask]), off


def slot_values(vals32):
    return pack([rlp_trimmed(vals32)])


def account_values(nonce, bal, sroot, code):
    """rlp([nonce, balance, storageRoot, codeHash]) per account (the payload is 68..108 bytes: a two-byte list header)"""
    n = len(nonce)
    nb, ns = rlp_trimmed(nonce.astype(">u8").view(np.uint8).reshape(n, 8)), rlp_trimmed(bal)
    plen = (9 - nb[1]) + (33 - ns[1]) + 66
    head = np.stack([np.full(n, 0xf8, np.uint8), plen.astype(np.uint8)], axis=1)
    h32 = lambda x: (np.concatenate([np.full((n, 1), 0xa0, np.uint8), x], axis=1), np.zeros(n, np.int64))  # noqa: E731
    return pack([(head, np.zeros(n, np.int64)), nb, ns, h32(sroot), h32(code)])


def node_csr(p):
    return p["nodes"], p["node_off"]


class Batch:
    """ranges for one verify call, built from range results"""

    def __init__(self):
        self.roots, self.origins, self.flags, self.counts, self.keys, self.vals, self.more = [], [], [], [], [], [], []

    def add(self, root, origin, keys, vals_off, whole, more):
        self.roots.append(root); self.origins.append(origin); self.flags.append(gpu.RANGE_WHOLE if whole else 0)
        self.counts.append(len(keys)); self.keys.append(keys); self.vals.append(vals_off); self.more.append(bool(more))

    def arrays(self):
        first = np.zeros(len(self.counts) + 1, np.uint64)
        first[1:] = np.cumsum(self.counts)
        keys = np.ascontiguousarray(np.concatenate(self.keys)) if self.keys else np.zeros((0, 32), np.uint8)
        data = np.concatenate([v for v, _ in self.vals]) if self.vals else np.zeros(1, np.uint8)
        offs, base = [np.zeros(1, np.uint64)], 0
        for v, o in self.vals:
            offs.append(o[1:] + np.uint64(base))
            base += int(o[-1])
        return (np.frombuffer(b"".join(self.roots), np.uint8), np.frombuffer(b"".join(self.origins), np.uint8), first, keys,
                np.concatenate([data, np.zeros(1, np.uint8)]), np.concatenate(offs), np.array(self.flags, np.uint8))


def account_batch(st, root, origins, per):
    r, _ = st.range([(o, ALL, per) for o in origins])
    b, prove = Batch(), []
    f = r["account_first"]
    for i, o in enumerate(origins):
        a, e = int(f[i]), int(f[i + 1])
        vals = account_values(r["nonce"][a:e], r["balance32"][a:e], r["storage_root32"][a:e], r["code_hash32"][a:e])
        b.add(root, o, r["account_keys32"][a:e], vals, False, r["account_more"][i])
        prove += [o] + ([r["account_keys32"][e - 1].tobytes()] if e > a else [])
    return b, st.prove(np.frombuffer(b"".join(dict.fromkeys(prove)), np.uint8))  # two ranges can end at the trie's last key


def storage_batch(st, accts, origins, per):
    """storage ranges of `accts` from `origins`: a complete trie (origin 0, nothing after) is WHOLE, the others proven"""
    r, _ = st.range(storage_ranges=[(a, o, ALL, per) for a, o in zip(accts, origins)])
    rd, _ = st.read(np.frombuffer(b"".join(accts), np.uint8))
    b, sacc, skeys = Batch(), [], []
    f = r["slot_first"]
    for i, (ak, o) in enumerate(zip(accts, origins)):
        a, e = int(f[i]), int(f[i + 1])
        more = bool(r["slot_more"][i])
        whole = o == ZERO and not more
        b.add(rd["storage_root32"][i].tobytes(), o, r["slot_keys32"][a:e], slot_values(r["slot_vals32"][a:e]), whole, more)
        if not whole:
            ks = list(dict.fromkeys([o] + ([r["slot_keys32"][e - 1].tobytes()] if e > a else [])))
            sacc += [i] * len(ks)
            skeys += ks
    p = st.prove(np.frombuffer(b"".join(accts), np.uint8), np.array(sacc, np.uint32) if sacc else None,
                 np.frombuffer(b"".join(skeys), np.uint8) if skeys else None)
    return b, p, r


def verify(ctx, b, p):
    roots, origins, first, keys, vals, voff, flags = b.arrays()
    nodes, noff = node_csr(p)
    ctx.synchronize()
    ctx.reset_stats()
    t0 = time.perf_counter()
    status, more = ctx.verify_ranges(nodes, noff, roots, origins, first, keys, vals, voff, flags)
    ms = (time.perf_counter() - t0) * 1e3
    s = ctx.stats()
    assert (status == 1).all(), np.unique(status, return_counts=True)
    assert [bool(x) for x in more] == b.more
    return dict(ms=ms, ranges=len(b.counts), entries=int(first[-1]), launches=s["launches"], h2d_bytes=s["h2d_bytes"],
                keccak_msgs=s["keccak_msgs"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every storage size (0.01 for a quick run)")
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--chunk", type=int, default=1 << 20)
    ap.add_argument("--full", type=int, default=1, help="whole-state verifications")
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    rng = np.random.default_rng(args.seed)
    gpu_name = card()
    akeys, nonce, bal, code, slot_acc, skeys, svals, store = build_state(rng, args.accounts, args.scale)
    ctx = gpu.Context(0)
    st = ctx.resident_state()
    root = st.apply(akeys, nonce, bal, code, None, slot_acc, skeys, svals)
    del slot_acc, skeys, svals
    rich = [akeys[a].tobytes() for a in sorted(store) if len(store[a].k)]
    rk = lambda: rng.integers(0, 256, 32, dtype=np.uint8).tobytes()  # noqa: E731
    med = lambda rows: {k: round(float(np.median([x[k] for x in rows])), 4) for k in rows[0]}  # noqa: E731
    out = {"gpu": gpu_name, "accounts": args.accounts, "slots": int(st.info()["n_slots"])}
    for name, make in (("snap_accounts", lambda: account_batch(st, root, [rk() for _ in range(64)], 5000)),
                       ("snap_storage", lambda: storage_batch(st, [rich[int(i)] for i in rng.choice(len(rich), 100, replace=False)],
                                                             [ZERO] * 99 + [rk()], 1000)[:2])):
        rows = []
        for c in range(args.warmup + args.calls):
            b, p = make()
            row = verify(ctx, b, p)
            if c >= args.warmup:
                rows.append(row)
        m = med(rows)
        out[name] = {"calls": len(rows), "median": m, "entries_per_s": round(m["entries"] / (m["ms"] / 1e3))}
    for run in range(args.full):
        rows, origin = [], ZERO
        while True:  # the accounts, one range per call
            b, p = account_batch(st, root, [origin], args.chunk)
            rows.append(verify(ctx, b, p))
            if not b.more[0]:
                break
            origin = (int.from_bytes(b.keys[0][-1].tobytes(), "big") + 1).to_bytes(32, "big")
        pending = [(a, ZERO) for a in rich]
        while pending:  # every account's slots, many accounts per call
            batch, pending = pending[:4096], pending[4096:]
            each = max(args.chunk // len(batch), 1)
            b, p, r = storage_batch(st, [a for a, _ in batch], [o for _, o in batch], each)
            rows.append(verify(ctx, b, p))
            for i, (a, _) in enumerate(batch):
                if b.more[i]:
                    pending.append((a, (int.from_bytes(b.keys[i][-1].tobytes(), "big") + 1).to_bytes(32, "big")))
        tot = {k: sum(x[k] for x in rows) for k in ("ms", "entries", "launches", "h2d_bytes", "keccak_msgs")}
        assert tot["entries"] == args.accounts + out["slots"], (tot, out["slots"])
        out["full"] = dict(calls=len(rows), **{k: round(v, 3) for k, v in tot.items()}, entries_per_s=round(tot["entries"] / (tot["ms"] / 1e3)))
    out["all_checked"] = True
    print(json.dumps(out))
    st.close()
    ctx.close()


if __name__ == "__main__":
    main()
