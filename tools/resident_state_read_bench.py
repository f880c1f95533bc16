"""Account and slot reads from the resident world state (phant_gpu_resident_state_read), now and 64 blocks back.

The state and the blocks are those of tools/resident_state_bench.py: 1,000,000 accounts and about 10M slots; 64 blocks
(3,000 accounts, 15,000 slot writes each) are applied with a journal of 64, so that back = 64 walks every record.  Request
shapes, each timed at back 0 and back 64:

  rpc     one account with storage and four of its slots (one absent) per call, many calls (eth_getBalance /
          eth_getStorageAt as an RPC node serves them); prove's call of the same shape is timed at back 0 for comparison
  block   3,000 accounts and 15,000 slots in one call (the pre-state reads of one block)
  batch   1,000,000 account reads and 1,000,000 slot reads in one call, reported as reads/s

Every request is drawn before the blocks, with the values it has then; after them its values now come from the host's copy
of the state.  Every value read is checked against the copy of its root (storage roots at back 0 against prove's).  Times
are host wall clock around the synchronous calls.  Also reported: the median apply at depth 64.  Prints one JSON line with
the card's name and power limit read in the same run.

    python tools/resident_state_read_bench.py [--accounts 1000000] [--scale 1.0] [--calls 200] [--blocks 8] [--batches 3]
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
from resident_state_bench import build_state, card, make_block, rand_rows  # noqa: E402


def groups(acc):
    """(account, the positions holding it) for each distinct account of acc"""
    o = np.argsort(acc, kind="stable")
    u, first = np.unique(acc[o], return_index=True)
    return zip((int(a) for a in u), np.split(o, first[1:]))


def lookup(store, acc, keys):
    """slot values of (account acc[j], keys[j]) in the host's copy (zero where absent)"""
    out = np.zeros((len(acc), 32), np.uint8)
    for a, j in groups(acc):
        s = store.get(a)
        if s is None or not len(s.k):
            continue
        ks, q = s.k.view("S32").ravel(), keys[j].view("S32").ravel()
        pos = np.minimum(np.searchsorted(ks, q), len(ks) - 1)
        hit = ks[pos] == q
        out[j[hit]] = s.v[pos[hit]]
    return out


class Request:
    """accounts (indices into the state) and slots (request account, key), with the values of the state when drawn"""

    def __init__(self, store, nonce, bal, code, accounts, slot_index, skeys):
        self.acc, self.sa, self.sk = np.asarray(accounts, np.int64), np.asarray(slot_index, np.uint32), np.ascontiguousarray(skeys)
        self.then = self.values(store, nonce, bal, code)

    def values(self, store, nonce, bal, code):
        return dict(nonce=nonce[self.acc].copy(), balance32=bal[self.acc].copy(), code_hash32=code[self.acc].copy(),
                    slot_vals32=lookup(store, self.acc[self.sa], self.sk))


def check(r, want):
    assert (r["account_status"] == 1).all()
    for f in ("nonce", "balance32", "code_hash32", "slot_vals32"):
        assert np.array_equal(r[f], want[f]), f
    assert np.array_equal(r["slot_status"], np.where(want["slot_vals32"].any(axis=1), 1, 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every storage size (0.01 for a quick run)")
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--blocks", type=int, default=8, help="block-shaped calls")
    ap.add_argument("--batches", type=int, default=3, help="1M + 1M calls")
    ap.add_argument("--batch", type=int, default=1_000_000)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    rng = np.random.default_rng(args.seed)
    gpu_name = card()
    na = args.accounts
    akeys, nonce, bal, code, slot_acc, skeys, svals, store = build_state(rng, na, args.scale)
    with_storage = np.array(sorted(store), np.int64)
    small = with_storage[with_storage >= 31]

    # ---- requests, drawn before the blocks ----
    def held(a, n):
        k = store[a].k
        return k[rng.choice(len(k), min(n, len(k)), replace=False)]

    rpc = []
    for _ in range(args.warmup + args.calls):
        a = int(with_storage[int(rng.integers(0, len(with_storage)))])
        sk = np.concatenate([held(a, 3), rand_rows(rng, 1)])
        rpc.append(Request(store, nonce, bal, code, [a], np.zeros(len(sk), np.uint32), sk))
    blocks = []
    for _ in range(args.warmup + args.blocks):
        rich = [int(x) for x in rng.choice(np.arange(0, 31), 6, replace=False)] + [int(x) for x in rng.choice(small, 994, replace=False)]
        accs = rich + [int(x) for x in rng.choice(np.arange(50_031, na), 2000, replace=False)]
        sk = np.concatenate([held(a, 15) for a in rich])[:15_000]
        si = np.repeat(np.arange(len(rich), dtype=np.uint32), [min(15, len(store[a].k)) for a in rich])[:15_000]
        blocks.append(Request(store, nonce, bal, code, accs, si, sk))
    nb = args.batch
    b_acc = rng.permutation(na)[:nb]
    rich = with_storage[np.isin(with_storage, b_acc)]
    b_slot_acc = rich[rng.integers(0, len(rich), nb)]
    b_sk = np.empty((nb, 32), np.uint8)
    for a, j in groups(b_slot_acc):
        k = store[a].k
        b_sk[j] = k[rng.integers(0, len(k), len(j))]
    where = np.empty(na, np.uint32)
    where[b_acc] = np.arange(nb, dtype=np.uint32)
    batch = Request(store, nonce, bal, code, b_acc, where[b_slot_acc], b_sk)
    ctx = gpu.Context(0)
    st = ctx.resident_state()
    st.apply(akeys, nonce, bal, code, None, slot_acc, skeys, svals)
    del slot_acc, skeys, svals

    # ---- 64 blocks with a journal of 64 ----
    st.set_journal(64)
    apply_ms = []
    for _ in range(64):
        touched, _, slot_index, sk, sv = make_block(rng, store, small, na, nonce, bal)
        ak = np.ascontiguousarray(akeys[touched])
        ctx.synchronize()
        t0 = time.perf_counter()
        st.apply(ak, nonce[touched], np.ascontiguousarray(bal[touched]), np.ascontiguousarray(code[touched]), None, slot_index, sk, sv)
        apply_ms.append((time.perf_counter() - t0) * 1e3)
    info = st.info()
    assert info["journal_applies"] == 64
    for q in rpc + blocks + [batch]:
        q.now = q.values(store, nonce, bal, code)
        q.ak = np.ascontiguousarray(akeys[q.acc])

    def timed(f):
        ctx.synchronize()
        ctx.reset_stats()
        t0 = time.perf_counter()
        out = f()
        return out, (time.perf_counter() - t0) * 1e3, ctx.stats()

    def leg(reqs, back, warm):
        rows = []
        for c, q in enumerate(reqs):
            (r, _), ms, s = timed(lambda: st.read(q.ak, q.sa, q.sk, back=back))
            check(r, q.now if back == 0 else q.then)
            assert s["keccak_msgs"] == 0 and s["launches"] <= 2, s
            if c >= warm:
                rows.append(dict(ms=ms, launches=s["launches"], h2d_bytes=s["h2d_bytes"], d2h_bytes=s["d2h_bytes"]))
        return rows

    med = lambda rows: {k: round(float(np.median([x[k] for x in rows])), 4) for k in rows[0]}  # noqa: E731
    p99 = lambda rows: round(float(np.percentile([x["ms"] for x in rows], 99)), 4)  # noqa: E731
    out = {"gpu": gpu_name, "accounts": na, "slots": int(info["n_slots"]), "journal_applies": 64,
           "apply_depth64_median_ms": round(float(np.median(apply_ms[8:])), 3)}
    for back in (0, 64):
        r = leg(rpc, back, args.warmup)
        out[f"rpc_back{back}"] = {"calls": len(r), "median": med(r), "p99_ms": p99(r)}
        r = leg(blocks, back, args.warmup)
        out[f"block_back{back}"] = {"calls": len(r), "median": med(r)}
        r = leg([batch] * (1 + args.batches), back, 1)
        m = med(r)
        out[f"batch_back{back}"] = {"calls": len(r), "median": m, "reads_per_s": round(2 * nb / (m["ms"] / 1e3))}
    # prove's RPC shape, at back 0, for comparison; its storage roots pin the read's
    rows = []
    for c, q in enumerate(rpc):
        p, ms, s = timed(lambda: st.prove(q.ak, q.sa, q.sk))
        r, _ = st.read(q.ak, q.sa, q.sk)
        assert np.array_equal(r["storage_root32"], p["storage_root32"]) and np.array_equal(r["slot_vals32"], p["slot_vals32"])
        if c >= args.warmup:
            rows.append(dict(ms=ms, launches=s["launches"]))
    out["prove_rpc_back0"] = {"calls": len(rows), "median": med(rows), "p99_ms": p99(rows)}
    out["all_values_checked"] = True
    print(json.dumps(out))
    st.close()


if __name__ == "__main__":
    main()
