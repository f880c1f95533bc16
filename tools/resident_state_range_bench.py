"""Account and storage ranges from the resident world state (phant_gpu_resident_state_range), now and 64 blocks back.

The state and the blocks are those of tools/resident_state_bench.py: 1,000,000 accounts and about 10M slots; 64 blocks
(3,000 accounts, 15,000 slot writes each) are applied with a journal of 64, so that back = 64 merges every record.  Request
shapes, each timed at back 0 and back 64:

  snap    one account range of 5,000 entries and 100 storage ranges of up to 1,000 slots in one call (a GetAccountRange
          and a GetStorageRanges as a snap server answers them, without the proofs)
  rpc     one storage range of 256 slots (debug_storageRangeAt)
  dump    the whole state in calls of at most 1M entries: the accounts range by range, then the slots of every account
          with storage, many accounts per call; reported as entries/s and PCIe bytes moved

Every entry returned is checked against the host's copy of the state at that root (keys, nonce, balance, codeHash, slot
values; the host copy holds no storage roots).  Times are host wall clock around the synchronous calls (the dump: around its
calls, without the checks).  Launches, H2D / D2H bytes and Keccak messages come from phant_gpu_stats.  Prints one JSON line
with the card's name and power limit read in the same run.

    python tools/resident_state_range_bench.py [--accounts 1000000] [--scale 1.0] [--calls 50] [--dumps 2]
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

ZERO, ALL = bytes(32), b"\xff" * 32


class Snapshot:
    """the host's copy of the state at one root: accounts sorted by key, each account's sorted slots"""

    def __init__(self, akeys, nonce, bal, code, store):
        o = np.argsort(akeys.view("S32").ravel(), kind="stable")
        self.order, self.keys = o, akeys.view("S32").ravel()[o]
        self.nonce, self.bal, self.code = nonce[o].copy(), bal[o].copy(), code[o].copy()
        self.slots = {akeys[a].tobytes(): (s.k, s.v.copy()) for a, s in store.items() if len(s.k)}

    def accounts(self, origin, limit, mx):
        a = np.searchsorted(self.keys, np.frombuffer(origin, "S32"))[0]
        b = np.searchsorted(self.keys, np.frombuffer(limit, "S32"), side="right")[0]
        return slice(a, min(b, a + mx)), b - a > mx

    def storage(self, akey, origin, limit, mx):
        k, v = self.slots.get(akey, (np.zeros((0, 32), np.uint8), np.zeros((0, 32), np.uint8)))
        ks = k.view("S32").ravel()
        a = np.searchsorted(ks, np.frombuffer(origin, "S32"))[0]
        b = np.searchsorted(ks, np.frombuffer(limit, "S32"), side="right")[0]
        e = min(b, a + mx)
        return k[a:e], v[a:e], b - a > mx


def check(r, snap, aranges, sranges):
    for i, (o, lim, mx) in enumerate(aranges):
        s, more = snap.accounts(o, lim, mx)
        a, b = int(r["account_first"][i]), int(r["account_first"][i + 1])
        assert bool(r["account_more"][i]) == more
        assert np.array_equal(r["account_keys32"][a:b].view("S32").ravel(), snap.keys[s])
        assert np.array_equal(r["nonce"][a:b], snap.nonce[s]) and np.array_equal(r["balance32"][a:b], snap.bal[s])
        assert np.array_equal(r["code_hash32"][a:b], snap.code[s])
    for j, (ak, o, lim, mx) in enumerate(sranges):
        k, v, more = snap.storage(ak, o, lim, mx)
        a, b = int(r["slot_first"][j]), int(r["slot_first"][j + 1])
        assert bool(r["slot_more"][j]) == more
        assert np.array_equal(r["slot_keys32"][a:b], k) and np.array_equal(r["slot_vals32"][a:b], v)


def dump(st, back, chunk):
    """the whole state in calls of at most `chunk` entries -> (account arrays, {account key: (slot keys, values)}, calls)"""
    parts, rich, origin, calls = [], [], ZERO, 0
    while True:
        r, _ = st.range([(origin, ALL, chunk)], back=back)
        calls += 1
        parts.append(r)
        k = r["account_keys32"]
        rich += [k[i].tobytes() for i in np.nonzero((r["storage_root32"] != EMPTY_ROOT).any(axis=1))[0]]
        if not r["account_more"][0]:
            break
        origin = (int.from_bytes(k[-1].tobytes(), "big") + 1).to_bytes(32, "big")
    slots, pending = {}, [(a, ZERO) for a in rich]
    while pending:
        batch, pending = pending[:chunk], pending[chunk:]
        each = max(chunk // len(batch), 1)
        r, _ = st.range(storage_ranges=[(a, o, ALL, each) for a, o in batch], back=back)
        calls += 1
        f = r["slot_first"]
        for i, (a, _) in enumerate(batch):
            k, v = r["slot_keys32"][f[i]:f[i + 1]], r["slot_vals32"][f[i]:f[i + 1]]
            slots.setdefault(a, []).append((k, v))
            if r["slot_more"][i]:
                pending.append((a, (int.from_bytes(k[-1].tobytes(), "big") + 1).to_bytes(32, "big")))
    acc = {f: np.concatenate([p[f] for p in parts]) for f in ("account_keys32", "nonce", "balance32", "code_hash32")}
    return acc, {a: (np.concatenate([k for k, _ in x]), np.concatenate([v for _, v in x])) for a, x in slots.items()}, calls


EMPTY_ROOT = np.frombuffer(bytes.fromhex("56e81f171bcc55a6ff8345e692c0f86e5b48e01b996cadc001622fb5e363b421"), np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every storage size (0.01 for a quick run)")
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--dumps", type=int, default=2)
    ap.add_argument("--chunk", type=int, default=1 << 20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    rng = np.random.default_rng(args.seed)
    gpu_name = card()
    na = args.accounts
    akeys, nonce, bal, code, slot_acc, skeys, svals, store = build_state(rng, na, args.scale)
    small = np.array(sorted(store), np.int64)
    small = small[small >= 31]
    then = Snapshot(akeys, nonce, bal, code, store)
    ctx = gpu.Context(0)
    st = ctx.resident_state()
    st.apply(akeys, nonce, bal, code, None, slot_acc, skeys, svals)
    del slot_acc, skeys, svals
    st.set_journal(64)
    for _ in range(64):
        touched, _, slot_index, sk, sv = make_block(rng, store, small, na, nonce, bal)
        st.apply(np.ascontiguousarray(akeys[touched]), nonce[touched], np.ascontiguousarray(bal[touched]),
                 np.ascontiguousarray(code[touched]), None, slot_index, sk, sv)
    assert st.info()["journal_applies"] == 64
    now = Snapshot(akeys, nonce, bal, code, store)
    rich = [akeys[a].tobytes() for a in sorted(store) if len(store[a].k)]
    rk = lambda: rng.integers(0, 256, 32, dtype=np.uint8).tobytes()  # noqa: E731

    def snap_req():
        return [(rk(), ALL, 5000)], [(rich[int(i)], ZERO if i % 2 else rk(), ALL, 1000) for i in rng.choice(len(rich), 100, replace=False)]

    def rpc_req():
        return [], [(rich[int(rng.integers(0, len(rich)))], rk(), ALL, 256)]

    def timed(f):
        ctx.synchronize()
        ctx.reset_stats()
        t0 = time.perf_counter()
        out = f()
        return out, (time.perf_counter() - t0) * 1e3, ctx.stats()

    med = lambda rows: {k: round(float(np.median([x[k] for x in rows])), 4) for k in rows[0]}  # noqa: E731
    out = {"gpu": gpu_name, "accounts": na, "slots": int(st.info()["n_slots"]), "journal_applies": 64}
    for back, snap in ((0, now), (64, then)):
        for name, make in (("snap", snap_req), ("rpc", rpc_req)):
            rows = []
            for c in range(args.warmup + args.calls):
                ar, sr = make()
                (r, _), ms, s = timed(lambda: st.range(ar, sr, back=back))
                check(r, snap, ar, sr)
                assert s["keccak_msgs"] == 0, s
                if c >= args.warmup:
                    rows.append(dict(ms=ms, entries=int(r["account_first"][-1] + r["slot_first"][-1]), launches=s["launches"],
                                     h2d_bytes=s["h2d_bytes"], d2h_bytes=s["d2h_bytes"]))
            out[f"{name}_back{back}"] = {"calls": len(rows), "median": med(rows)}
        rows = []
        for c in range(1 + args.dumps):
            (acc, slots, calls), ms, s = timed(lambda: dump(st, back, args.chunk))
            assert s["keccak_msgs"] == 0, s
            assert np.array_equal(acc["account_keys32"].view("S32").ravel(), snap.keys)
            for f, want in (("nonce", snap.nonce), ("balance32", snap.bal), ("code_hash32", snap.code)):
                assert np.array_equal(acc[f], want), f
            assert slots.keys() == snap.slots.keys()
            for a, (k, v) in slots.items():
                assert np.array_equal(k, snap.slots[a][0]) and np.array_equal(v, snap.slots[a][1])
            entries = len(acc["nonce"]) + sum(len(k) for k, _ in slots.values())
            if c >= 1:
                rows.append(dict(ms=ms, calls=calls, entries=entries, launches=s["launches"], h2d_bytes=s["h2d_bytes"], d2h_bytes=s["d2h_bytes"]))
        m = med(rows)
        out[f"dump_back{back}"] = {"runs": len(rows), "median": m, "entries_per_s": round(m["entries"] / (m["ms"] / 1e3)),
                                   "pcie_bytes_per_s": round((m["h2d_bytes"] + m["d2h_bytes"]) / (m["ms"] / 1e3))}
    out["all_entries_checked"] = True
    print(json.dumps(out))
    st.close()


if __name__ == "__main__":
    main()
