"""Undo on the resident world state (phant_gpu_resident_state_set_journal / _revert), block after block.

The state and the blocks are those of tools/resident_state_bench.py: 1,000,000 accounts and about 10M slots; each block
touches 3,000 accounts and writes 15,000 slots.  Reported per block:

  apply depth 0    phant_gpu_resident_state_apply with no journal
  apply depth 64   the same with a journal of 64 (capturing the undo record); alternated with depth 0 block by block, in
                   one process, so that the difference is the capture's cost
  revert(1)        undoing the block just applied (then it is applied again)
  revert(8)        undoing the last 8 blocks at once (then they are applied again)
  reload           the alternative: a new resident state loaded with the whole current state from the host

Every root is checked: a revert must give back the root before the blocks it undoes, and applying a block again must give
the root it gave the first time; the reload must give the current root.  Times are host wall clock around the synchronous
calls.  Prints one JSON line per leg with the card's name and power limit.

    python tools/resident_state_revert_bench.py [--accounts 1000000] [--warmup 2] [--blocks 16] [--rounds8 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from phant_b200 import gpu  # noqa: E402
from resident_state_bench import build_state, card, make_block  # noqa: E402


def timed(f):
    t0 = time.perf_counter()
    r = f()
    return r, (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every storage size (0.01 for a quick run)")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--blocks", type=int, default=16, help="timed blocks of the alternating depth-0 / depth-64 leg")
    ap.add_argument("--rounds8", type=int, default=3, help="timed revert(8) rounds")
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    rng = np.random.default_rng(args.seed)
    gpu_name = card()
    na = args.accounts
    akeys, nonce, bal, code, slot_acc, skeys, svals, store = build_state(rng, na, args.scale)
    ns = len(skeys)
    ctx = gpu.Context(0)
    st = ctx.resident_state()
    st.apply(akeys, nonce, bal, code, None, slot_acc, skeys, svals)
    del slot_acc, skeys, svals
    with_storage = np.array(sorted(store), np.int64)
    small = with_storage[with_storage >= 31]

    def block():
        touched, _, slot_index, sk, sv = make_block(rng, store, small, na, nonce, bal)
        return (akeys[touched], nonce[touched].copy(), bal[touched].copy(), code[touched], None, slot_index, sk, sv)

    legs = {"apply_depth0": [], "apply_depth64": [], "revert1": [], "revert8": []}
    stats = {k: [] for k in legs}

    def rec(name, ms, warm):
        if not warm:
            legs[name].append(ms)
            stats[name].append(ctx.stats())

    # ---- apply at depth 0 and 64, alternated; after each depth-64 block, revert(1) and the same block again ----
    for b in range(args.warmup + 2 * args.blocks):
        warm = b < args.warmup
        depth = 64 if b % 2 else 0
        st.set_journal(depth)
        d = block()
        before = st.root()
        ctx.reset_stats()
        root, ms = timed(lambda: st.apply(*d))
        rec(f"apply_depth{depth}", ms, warm)
        if depth:
            ctx.reset_stats()
            back, ms = timed(lambda: st.revert(1))
            assert back == before and st.root() == before, f"block {b}: revert(1) did not give back the root before it"
            rec("revert1", ms, warm)
            assert st.apply(*d) == root, f"block {b}: the block applied again gave another root"

    # ---- revert(8): eight blocks at depth 64, undone at once, applied again ----
    st.set_journal(64)
    for r in range(1 + args.rounds8):
        before = st.root()
        ds = [block() for _ in range(8)]
        roots = [st.apply(*d) for d in ds]
        ctx.reset_stats()
        back, ms = timed(lambda: st.revert(8))
        assert back == before and st.root() == before, f"round {r}: revert(8) did not give back the root before the 8 blocks"
        rec("revert8", ms, r == 0)
        for d, want in zip(ds, roots):
            assert st.apply(*d) == want, f"round {r}: a block applied again gave another root"
    info = st.info()
    st.set_journal(0)

    # ---- the alternative to a revert: reload the whole current state ----
    live = sorted(store)
    sizes = np.zeros(na, np.int64)
    for a in live:
        sizes[a] = len(store[a].k)
    full_acc = np.repeat(np.arange(na, dtype=np.uint32), sizes)
    full_k = np.concatenate([store[a].k for a in live])
    full_v = np.concatenate([store[a].v for a in live])
    want = st.root()
    st.close()
    fresh = ctx.resident_state()
    ctx.reset_stats()
    got, reload_ms = timed(lambda: fresh.apply(akeys, nonce, bal, code, None, full_acc, full_k, full_v))
    assert got == want, "reload gave another root"
    fresh.close()

    for name, ms in legs.items():
        ms = np.array(ms)
        s = stats[name]
        print(json.dumps({"leg": name, "gpu": gpu_name, "accounts": na, "slots": ns, "samples": len(ms),
                          "ms_median": round(float(np.median(ms)), 3), "ms_min": round(float(ms.min()), 3),
                          "ms_max": round(float(ms.max()), 3), "launches": int(np.median([x["launches"] for x in s])),
                          "h2d_bytes": int(np.median([x["h2d_bytes"] for x in s])),
                          "keccak_msgs": int(np.median([x["keccak_msgs"] for x in s]))}))
    print(json.dumps({"leg": "reload", "gpu": gpu_name, "accounts": na, "slots": len(full_k), "ms": round(reload_ms, 1)}))
    print(json.dumps({"roots_agree": True, "device_bytes_depth64": info["device_bytes"], "journal_bytes_depth64": info["journal_bytes"],
                      "gpu": gpu_name}))
    ctx.close()


if __name__ == "__main__":
    main()
