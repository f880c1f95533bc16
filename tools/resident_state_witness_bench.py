"""Execution witnesses from the resident world state (phant_gpu_resident_state_witness), block after block.

The state and the blocks are those of tools/resident_state_bench.py: 1,000,000 accounts and about 10M slots; each block
touches 3,000 accounts and writes 15,000 slots.  For each block, on the state before it:

  witness   phant_gpu_resident_state_witness + _copy (the node set to the host)
  T         phant_gpu_transition_roots on that node set, the state's root and the block's diff
  apply     phant_gpu_resident_state_apply, which moves the state to the next block

Host wall clock around each synchronous call.  Every T root must equal the apply root.  Reported: medians of ms per call,
and for the witness its launches, H2D / D2H bytes, Keccak messages, nodes and bytes, with the card's name and power limit
read in the same run.

    python tools/resident_state_witness_bench.py [--accounts 1000000] [--scale 1.0] [--blocks 8] [--warmup 2]
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
from resident_state_bench import build_state, card, make_block  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every storage size (0.01 for a quick run)")
    ap.add_argument("--blocks", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    rng = np.random.default_rng(args.seed)
    gpu_name = card()
    na = args.accounts
    akeys, nonce, bal, code, slot_acc, skeys, svals, store = build_state(rng, na, args.scale)
    ctx = gpu.Context(0)
    st = ctx.resident_state()
    st.apply(akeys, nonce, bal, code, None, slot_acc, skeys, svals)
    del slot_acc, skeys, svals
    with_storage = np.array(sorted(store), np.int64)
    small = with_storage[with_storage >= 31]

    def timed(f):
        ctx.synchronize()
        ctx.reset_stats()
        t0 = time.perf_counter()
        out = f()
        return out, (time.perf_counter() - t0) * 1e3, ctx.stats()

    rows = []
    for b in range(args.warmup + args.blocks):
        touched, _, slot_index, sk, sv = make_block(rng, store, small, na, nonce, bal)
        d = dict(account_keys32=akeys[touched], nonce=nonce[touched].copy(), balance32=bal[touched].copy(), code_hash32=code[touched],
                 slot_account=slot_index, slot_keys32=sk, slot_vals32=sv)
        pre = np.frombuffer(st.root(), np.uint8)
        (nodes, off), w_ms, w_stats = timed(lambda: st.witness(**d))
        (roots, status), t_ms, _ = timed(lambda: ctx.transition_roots(nodes, off, pre, **d))
        root, a_ms, _ = timed(lambda: st.apply(**d))
        assert status[0] == 1 and roots[0].tobytes() == root, b
        if b >= args.warmup:
            rows.append(dict(witness_ms=w_ms, t_ms=t_ms, apply_ms=a_ms, launches=w_stats["launches"], h2d_bytes=w_stats["h2d_bytes"],
                             d2h_bytes=w_stats["d2h_bytes"], keccak_msgs=w_stats["keccak_msgs"], nodes=len(off) - 1, bytes=int(off[-1])))
    med = {k: float(np.median([r[k] for r in rows])) for k in rows[0]}
    print(json.dumps({"gpu": gpu_name, "accounts": na, "scale": args.scale, "blocks": len(rows), "median": {k: round(v, 3) for k, v in med.items()},
                      "t_roots_equal_apply_roots": True}))
    st.close()


if __name__ == "__main__":
    main()
