"""Contract code beside the resident world state (phant_gpu_resident_state_put_codes / _codes / _prune_codes).

The state is that of tools/resident_state_bench.py (1,000,000 accounts, about 10M slots) with seeded contract code: --codes
distinct codes whose lengths are drawn from a seeded log-normal distribution (median about 3 KB) capped at 24,576 B, spread
over --share of the accounts; the other accounts have no code.  64 blocks of that tool's shape (3,000 accounts, 15,000 slot
writes) are applied with a journal of 64, each after a put of its own 20 new codes, which 20 of its accounts take.  Timed:

  put_load     the whole load's codes into an empty store (codes/s, GB/s hashed and stored)
  put_block    one block's 20 new codes
  codes_rpc    one hash (eth_getCode)
  codes_snap   distinct held hashes up to about 512 KB of code (snap GetByteCodes)
  codes_wit    the distinct codes of a 3,000-account block's accounts (an execution witness's `codes`)
  get_code     1,000 accounts at back 0 and at back 64: read, then codes
  prune        at journal depth 64
  apply        the median apply at depth 64, with an empty store and with the full one, alternately

Every code returned is checked against the host's copy.  Times are host wall clock around the synchronous calls; launches,
H2D / D2H bytes and Keccak messages come from phant_gpu_stats.  --apply-only (with --tree, another built checkout's
phant_b200 package, e.g. the parent commit's) times only the apply, so that two builds can be run alternately.  Prints one
JSON line with the card's name and power limit read in the same run.

    python tools/resident_state_code_bench.py [--accounts 1000000] [--scale 1.0] [--codes 50000] [--share 0.2]
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
from resident_state_bench import build_state, card, make_block  # noqa: E402

gpu = None  # phant_b200.gpu, imported by main() from the tree --tree names
EMPTY_CODE_HASH = np.frombuffer(bytes.fromhex("c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470"), np.uint8)


def seeded_codes(rng, n):
    lens = np.clip(rng.lognormal(8.0, 1.0, n), 1, 24_576).astype(np.int64)
    return [rng.bytes(int(x)) for x in lens]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every storage size (0.01 for a quick run)")
    ap.add_argument("--codes", type=int, default=50_000)
    ap.add_argument("--share", type=float, default=0.2)
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--apply-blocks", type=int, default=10, help="apply pairs (empty store, full store) timed after the journal fills")
    ap.add_argument("--apply-only", action="store_true", help="time only the apply at depth 64 (no code call: any build)")
    ap.add_argument("--tree", default=None, help="import phant_b200 (and its built library) from this checkout instead")
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    if args.tree:
        sys.path.insert(0, os.path.abspath(args.tree))
    global gpu
    from phant_b200 import gpu
    rng = np.random.default_rng(args.seed)
    gpu_name = card()
    na = args.accounts
    akeys, nonce, bal, code, slot_acc, skeys, svals, store = build_state(rng, na, args.scale)
    ctx = gpu.Context(0)

    def timed(f):
        ctx.synchronize()
        ctx.reset_stats()
        t0 = time.perf_counter()
        out = f()
        return out, (time.perf_counter() - t0) * 1e3, ctx.stats()

    med = lambda rows: {k: round(float(np.median([x[k] for x in rows])), 4) for k in rows[0]}  # noqa: E731
    out = {"gpu": gpu_name, "accounts": na}
    held = {}  # hash -> code
    if not args.apply_only:
        pool = seeded_codes(rng, args.codes)
        warm = ctx.resident_state()
        warm.put_codes(pool[:1000])
        warm.close()
        st_probe = ctx.resident_state()
        hashes, ms, s = timed(lambda: st_probe.put_codes(pool))
        st_probe.close()
        nbytes = sum(map(len, pool))
        out["put_load"] = {"codes": len(pool), "bytes": nbytes, "ms": round(ms, 3), "codes_per_s": round(len(pool) / (ms / 1e3)),
                           "gb_per_s": round(nbytes / (ms / 1e3) / 1e9, 3), "launches": s["launches"], "h2d_bytes": s["h2d_bytes"]}
        held = {h.tobytes(): c for h, c in zip(hashes, pool)}
        with_code = rng.random(na) < args.share
        code[:] = EMPTY_CODE_HASH
        code[with_code] = hashes[rng.integers(0, len(pool), int(with_code.sum()))]
    then_code = code.copy()
    st = ctx.resident_state()
    if not args.apply_only:
        st.put_codes(pool)
    st.apply(akeys, nonce, bal, code, None, slot_acc, skeys, svals)
    del slot_acc, skeys, svals
    st.set_journal(64)
    small = np.array(sorted(store), np.int64)
    small = small[small >= 31]
    rows = []
    for b in range(64):
        touched, _, slot_index, sk, sv = make_block(rng, store, small, na, nonce, bal)
        if not args.apply_only:
            new = seeded_codes(rng, 20)
            nh, ms, s = timed(lambda: st.put_codes(new))
            held.update((h.tobytes(), c) for h, c in zip(nh, new))
            code[touched[-20:]] = nh
            if b >= args.warmup:
                rows.append(dict(ms=ms, launches=s["launches"], h2d_bytes=s["h2d_bytes"], keccak_msgs=s["keccak_msgs"]))
        st.apply(np.ascontiguousarray(akeys[touched]), nonce[touched], np.ascontiguousarray(bal[touched]), np.ascontiguousarray(code[touched]),
                 None, slot_index, sk, sv)
    assert st.info()["journal_applies"] == 64
    if rows:
        out["put_block"] = {"calls": len(rows), "median": med(rows)}

    def codes_checked(q):
        (status, got), ms, s = timed(lambda: st.codes(np.frombuffer(b"".join(q), np.uint8)))
        assert (status == 1).all() and got == [held.get(h, b"") for h in q]
        assert s["keccak_msgs"] == 0, s
        return dict(ms=ms, hashes=len(q), bytes=sum(map(len, got)), launches=s["launches"], d2h_bytes=s["d2h_bytes"])

    if not args.apply_only:
        hl = list(held)
        shapes = {"codes_rpc": lambda: [hl[int(rng.integers(0, len(hl)))]]}

        def snap():
            q, tot = [], 0
            for i in rng.permutation(len(hl)):
                q.append(hl[int(i)])
                tot += len(held[hl[int(i)]])
                if tot >= 512 * 1024:
                    return q
            return q

        def wit():
            touched = rng.choice(na, 3000, replace=False)
            return sorted({code[a].tobytes() for a in touched} - {EMPTY_CODE_HASH.tobytes()})
        shapes["codes_snap"], shapes["codes_wit"] = snap, wit
        for name, make in shapes.items():
            rr = [codes_checked(make()) for _ in range(args.warmup + args.calls)][args.warmup:]
            out[name] = {"calls": len(rr), "median": med(rr)}
        for back, ch in ((0, code), (64, then_code)):
            rr = []
            for c in range(args.warmup + args.calls):
                pick = rng.choice(na, 1000, replace=False)

                def get_code():
                    r, _ = st.read(np.ascontiguousarray(akeys[pick]), back=back)
                    return st.codes(np.where(r["account_status"][:, None] == 1, r["code_hash32"], EMPTY_CODE_HASH))
                (status, got), ms, s = timed(get_code)
                assert (status == 1).all() and got == [held.get(ch[a].tobytes(), b"") for a in pick], back
                if c >= args.warmup:
                    rr.append(dict(ms=ms, bytes=sum(map(len, got)), launches=s["launches"]))
            out[f"get_code_back{back}"] = {"calls": len(rr), "median": med(rr)}
        rr = []
        for c in range(1 + args.calls // 5):
            _, ms, s = timed(st.prune_codes)
            assert s["keccak_msgs"] == 0, s
            if c >= 1:
                rr.append(dict(ms=ms, launches=s["launches"]))
        i = st.info()
        out["prune"] = {"calls": len(rr), "median": med(rr), "n_codes": i["n_codes"], "code_bytes": i["code_bytes"]}
        q = list(held)[:2000]
        status, got = st.codes(np.frombuffer(b"".join(q), np.uint8))
        assert all(g == held[h] for s_, g, h in zip(status, got, q) if s_ == 1)

    # ---- apply at depth 64: with the full store, and (alternately) with an empty one ----
    empty = ctx.resident_state() if not args.apply_only else None
    legs = {"full": [], "empty": []} if not args.apply_only else {"store": []}
    if empty is not None:  # a twin with no code: the same tables through a second load
        _, _, _, _, sa2, sk2, sv2, _ = build_state(np.random.default_rng(args.seed), na, args.scale)
        empty.apply(akeys, nonce, bal, code, None, sa2, sk2, sv2)
        del sa2, sk2, sv2
        empty.set_journal(64)
    for b in range(args.warmup + args.apply_blocks):
        touched, _, slot_index, sk, sv = make_block(rng, store, small, na, nonce, bal)
        arrays = (np.ascontiguousarray(akeys[touched]), nonce[touched], np.ascontiguousarray(bal[touched]), np.ascontiguousarray(code[touched]),
                  None, slot_index, sk, sv)
        for name, s_ in (((("full", st), ("empty", empty)) if empty is not None else (("store", st),))):
            _, ms, s = timed(lambda: s_.apply(*arrays))
            if b >= args.warmup:
                legs[name].append(dict(ms=ms, launches=s["launches"]))
    for name, rr in legs.items():
        out[f"apply_depth64_{name}"] = {"blocks": len(rr), "median": med(rr)}
    out["all_codes_checked"] = not args.apply_only
    print(json.dumps(out))
    st.close()
    if empty is not None:
        empty.close()


if __name__ == "__main__":
    main()
