"""Snap range answers (GetAccountRange / GetStorageRanges) from the resident world state (phant_gpu_resident_state_snap_ranges
+ _copy), against the composition they replace.

The state is that of tools/resident_state_bench.py: 1,000,000 accounts and about 10M slots.  Calls of 1, 16 and 128 requests
at 512 KiB (geth's syncer request size) and at 2 MiB, of two kinds:

  account   requests from random origins
  storage   requests of 64 accounts with storage (the 2M- and 100k-slot accounts among them), from origin 0

The composition is what a server did before: `range` with max = bytes / 37 + 1 (storage: hard / 33 + 1 per account), the
byte cut and slim encoding on the host, then one `prove` for the boundary proofs; it is timed in the same run, alternated
call by call with snap_ranges.  Host wall clock around each synchronous call, copies to the host included.  Reported per
shape: median and p99 ms per call, answer MB/s (entries' keys and bodies plus proof bytes), launches, H2D and D2H bytes of
a call, and the card's name and power limit read in the same run.

    python tools/resident_state_snap_bench.py [--accounts 1000000] [--scale 1.0] [--calls 20] [--warmup 2]
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
from phant_b200.host import EMPTY_CODE_HASH, EMPTY_MPT_ROOT, _rlp_list, _rlp_str, _rlp_uint  # noqa: E402
from resident_state_bench import build_state, card  # noqa: E402

FF = b"\xff" * 32


def slim(nonce, bal32, sroot, code):
    return _rlp_list([_rlp_uint(int(nonce)), _rlp_uint(int.from_bytes(bal32, "big")), _rlp_str(b"" if sroot == EMPTY_MPT_ROOT else sroot),
                      _rlp_str(b"" if code == EMPTY_CODE_HASH else code)])


def composed(st, ar, sr):
    """the answers the way a server composed them before: range, a host cut with slim encoding, then prove; bytes returned"""
    total = 0
    if ar:
        r, _ = st.range([(o, lim, b // 37 + 1) for o, lim, b in ar])
        first, keys = r["account_first"], []
        for i, (o, _, b) in enumerate(ar):
            size = 0
            for e in range(int(first[i]), int(first[i + 1])):
                body = slim(r["nonce"][e], r["balance32"][e].tobytes(), r["storage_root32"][e].tobytes(), r["code_hash32"][e].tobytes())
                size += 32 + len(body)
                last = r["account_keys32"][e].tobytes()
                if size > b:
                    break
            keys += [o] + ([last] if size else [])
            total += size
        p = st.prove(np.frombuffer(b"".join(dict.fromkeys(keys)), np.uint8))
        total += int(p["nodes"].size)
    for accts, o, lim, b in sr:
        hard = b + b // 10
        r, _ = st.range(storage_ranges=[(a, o if i == 0 else bytes(32), lim if i == 0 else FF, hard // 33 + 1) for i, a in enumerate(accts)])
        first, size, proved = r["slot_first"], 0, None
        for i in range(len(accts)):
            if size >= b:
                break
            for e in range(int(first[i]), int(first[i + 1])):
                if size >= hard:
                    proved = (i, r["slot_keys32"][e - 1].tobytes())
                    break
                v = r["slot_vals32"][e].tobytes().lstrip(b"\x00")
                size += 32 + len(_rlp_str(v))
            if proved:
                break
        total += size
        if proved:
            p = st.prove(np.frombuffer(accts[proved[0]], np.uint8), np.zeros(2, np.uint32), np.frombuffer(bytes(32) + proved[1], np.uint8))
            total += int(p["nodes"].size)
    return total


def served(ans):
    n = sum(len(k) + len(b) for lst in ans["accounts"] for k, b in lst)
    n += sum(len(k) + len(b) for req in ans["slots"] for lst in req for k, b in lst)
    return n + sum(len(x) for p in ans["proofs"] for x in p)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every storage size (0.01 for a quick run)")
    ap.add_argument("--calls", type=int, default=20)
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
    rich = [akeys[a].tobytes() for a in sorted(store)]

    def shape(kind, n, nbytes):
        if kind == "account":
            return [(akeys[int(i)].tobytes(), FF, nbytes) for i in rng.integers(0, na, n)], []
        return [], [([rich[int(i)] for i in rng.choice(len(rich), 64, replace=False)], bytes(32), FF, nbytes) for _ in range(n)]

    def timed(f):
        ctx.synchronize()
        ctx.reset_stats()
        t0 = time.perf_counter()
        out = f()
        ms = (time.perf_counter() - t0) * 1e3
        return out, ms, ctx.stats()

    results = []
    for kind in ("account", "storage"):
        for n in (1, 16, 128):
            for nbytes in (512 << 10, 2 << 20):
                rows = {"snap_ranges": [], "composed": []}
                for c in range(args.warmup + args.calls):
                    ar, sr = shape(kind, n, nbytes)
                    ans, ms, s = timed(lambda: st.snap_ranges(ar, sr))
                    got, ms2, s2 = timed(lambda: composed(st, ar, sr))
                    if c >= args.warmup:
                        rows["snap_ranges"].append(dict(ms=ms, mb_s=served(ans) / ms / 1e3, launches=s["launches"], h2d_bytes=s["h2d_bytes"],
                                                        d2h_bytes=s["d2h_bytes"]))
                        rows["composed"].append(dict(ms=ms2, mb_s=got / ms2 / 1e3, launches=s2["launches"], h2d_bytes=s2["h2d_bytes"],
                                                     d2h_bytes=s2["d2h_bytes"]))
                out = {"kind": kind, "requests": n, "bytes": nbytes}
                for k, rs in rows.items():
                    med = {f: round(float(np.median([x[f] for x in rs])), 3) for f in rs[0]}
                    med["p99_ms"] = round(float(np.percentile([x["ms"] for x in rs], 99)), 3)
                    out[k] = med
                results.append(out)
                print(json.dumps(out), flush=True)
    print(json.dumps({"gpu": gpu_name, "accounts": na, "scale": args.scale, "calls": args.calls, "results": results}))
    st.close()


if __name__ == "__main__":
    main()
