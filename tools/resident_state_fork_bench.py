"""Forks of the resident world state (phant_gpu_resident_state_fork): a new state at a root the undo journal reaches.

The state and the blocks are those of tools/resident_state_bench.py: 1,000,000 accounts and about 10M slots, then 64 blocks
of 3,000 accounts (15,000 slot writes each) applied at journal depth 64.  Reported:

  fork(back)          for back in {0, 1, 8, 64}: median and p99 ms per call (host wall clock around the synchronous call),
                      each fork closed before the next; every fork's root is checked against read(back)'s
  trie_nodes          on fork(64): a 1,024-path request of account-trie paths at depths 0..8 (prefixes of random keys)
  account_range_proof on fork(64), through host.ResidentStateDB.fork: 256 accounts from a random origin with both boundary
                      proofs
  device_bytes        of the parent (with its journal) and of fork(0) and fork(64)

Launches and H2D / D2H bytes of each call come from the context's stats.  One JSON line per leg, with the card's name and
power limit read in the same run.

    python tools/resident_state_fork_bench.py [--accounts 1000000] [--scale 1.0] [--blocks 64] [--calls 20] [--calls64 8]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from phant_b200 import gpu, host  # noqa: E402
from resident_state_bench import build_state, card, make_block  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every storage size (0.01 for a quick run)")
    ap.add_argument("--blocks", type=int, default=64, help="blocks applied at journal depth 64 (the deepest fork)")
    ap.add_argument("--calls", type=int, default=20, help="timed forks per back below 64, and timed serving calls")
    ap.add_argument("--calls64", type=int, default=8, help="timed forks at the deepest back")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    rng = np.random.default_rng(args.seed)
    gpu_name = card()
    na = args.accounts
    akeys, nonce, bal, code, slot_acc, skeys, svals, store = build_state(rng, na, args.scale)
    ns = len(skeys)
    ctx = gpu.Context(0)
    rs = host.ResidentStateDB(ctx)
    st = rs.state
    st.apply(akeys, nonce, bal, code, None, slot_acc, skeys, svals)
    del slot_acc, skeys, svals
    with_storage = np.array(sorted(store), np.int64)
    small = with_storage[with_storage >= 31]
    rs.set_journal(64)
    for _ in range(args.blocks):
        touched, _, slot_index, sk, sv = make_block(rng, store, small, na, nonce, bal)
        st.apply(akeys[touched], nonce[touched].copy(), bal[touched].copy(), code[touched], None, slot_index, sk, sv)
    parent = st.info()
    deepest = min(64, args.blocks)
    want = {b: st.read(np.zeros(0, np.uint8), back=b)[1] for b in sorted({0, 1, 8, deepest}) if b <= deepest}

    def timed(f):
        ctx.synchronize()
        ctx.reset_stats()
        t0 = time.perf_counter()
        out = f()
        return out, (time.perf_counter() - t0) * 1e3, ctx.stats()

    def line(leg, rows, **extra):
        ms = np.array([r[0] for r in rows])
        s = [r[1] for r in rows]
        print(json.dumps({"leg": leg, "gpu": gpu_name, "accounts": na, "slots": ns, "samples": len(ms),
                          "ms_median": round(float(np.median(ms)), 3), "ms_p99": round(float(np.percentile(ms, 99)), 3),
                          "launches": int(np.median([x["launches"] for x in s])), "h2d_bytes": int(np.median([x["h2d_bytes"] for x in s])),
                          "d2h_bytes": int(np.median([x["d2h_bytes"] for x in s])), **extra}), flush=True)

    fork_bytes = {}
    for back, root in want.items():
        rows = []
        for c in range(args.warmup + (args.calls64 if back == deepest and back > 8 else args.calls)):
            f, ms, s = timed(lambda: st.fork(back))
            assert f.root() == root, f"fork({back}) is not at read({back})'s root"
            fork_bytes[back] = f.info()["device_bytes"]
            f.close()
            if c >= args.warmup:
                rows.append((ms, s))
        line(f"fork({back})", rows, device_bytes=fork_bytes[back])
    assert st.root() == want[0] and st.info() == parent, "a fork changed its parent"

    # ---- serving at the deepest root, from one fork ----
    fk = rs.fork(deepest)
    assert fk.state.root() == want[deepest]
    rows = []
    for c in range(args.warmup + args.calls):
        keys = akeys[rng.integers(0, na, 1024)]
        depth = rng.integers(0, 9, 1024)
        paths = np.zeros((1024, 32), np.uint8)
        for i, d in enumerate(depth):
            paths[i, :(d + 1) // 2] = keys[i, :(d + 1) // 2]
            if d & 1:
                paths[i, d // 2] &= 0xf0
        (status, blobs), ms, s = timed(lambda: fk.state.trie_nodes(paths, depth.astype(np.uint8)))
        assert (status[depth == 0] == 1).all()
        if c >= args.warmup:
            rows.append((ms, s))
    line(f"trie_nodes_1024_paths_at_fork({deepest})", rows)
    rows = []
    for c in range(args.warmup + args.calls):
        origin = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
        p, ms, s = timed(lambda: fk.account_range_proof(origin, host.MAX_KEY, 256))
        assert len(p["accounts"]) == 256 or not p["more"]
        if c >= args.warmup:
            rows.append((ms, s))
    line(f"account_range_proof_256_at_fork({deepest})", rows)
    ok, _ = host.verify_account_range(ctx, want[deepest], origin, p["accounts"], p["proof"])
    assert ok, "the last range answer from the fork does not verify against its root"
    fk.close()
    print(json.dumps({"roots_agree": True, "gpu": gpu_name, "parent_device_bytes": parent["device_bytes"],
                      "parent_journal_bytes": parent["journal_bytes"], "fork_device_bytes": {str(k): v for k, v in fork_bytes.items()}}))
    rs.close()
    ctx.close()


if __name__ == "__main__":
    main()
