"""Resident world state (phant_gpu_resident_state_*) against the best the kind-1 ABI can do, block after block.

Default shape: 1,000,000 accounts and about 10M slots -- one account with 2M slots, thirty with 100k, 50,000 with 100 and the
rest with none.  Each block touches 3,000 accounts and writes 15,000 slots (70% updates, 20% inserts, 10% deletes), 30 of them
in the 2M-slot account.  Slot values are 32 bytes with a non-zero first byte.

  resident   one phant_gpu_resident_state_apply per block with only the changed slots
  kind 1     one phant_gpu_mpt_roots call re-rooting every touched account's whole storage, then one phant_gpu_trie_update
             of the touched accounts' leaves (encoded on the host, not timed)

Both run in the same process, alternating block by block; the roots must agree on every block.  Times are host wall clock
around the synchronous calls.  Prints one JSON line per leg and the card's name and power limit beside the numbers.

    python tools/resident_state_bench.py [--accounts 1000000] [--warmup 3] [--blocks 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from phant_b200 import gpu  # noqa: E402

EMPTY_ROOT = bytes.fromhex("56e81f171bcc55a6ff8345e692c0f86e5b48e01b996cadc001622fb5e363b421")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def rand_rows(rng, n, width=32):
    return rng.integers(0, 256, (n, width), dtype=np.uint8)


def rand_vals(rng, n):
    v = rand_rows(rng, n)
    v[:, 0] = 1 + rng.integers(0, 255, n)  # 32-byte values: rlp = a0 || value
    return v


def rlp_bytes(b):
    b = b.lstrip(b"\x00")
    if len(b) == 1 and b[0] < 0x80:
        return b
    return bytes([0x80 + len(b)]) + b


def leaf(nonce, bal, sroot, code):
    body = rlp_bytes(int(nonce).to_bytes(8, "big")) + rlp_bytes(bal) + b"\xa0" + sroot + b"\xa0" + code
    return (bytes([0xc0 + len(body)]) if len(body) <= 55 else bytes([0xf8, len(body)])) + body


class Storage:
    """one account's storage, sorted by key ('S32' orders as bytes)"""

    def __init__(self, keys, vals):
        o = np.argsort(keys.view("S32").ravel(), kind="stable")
        self.k, self.v = keys[o], vals[o]

    def write(self, keys, vals):
        zero = ~vals.any(axis=1)
        ks = self.k.view("S32").ravel()
        q = keys.view("S32").ravel()
        pos = np.searchsorted(ks, q)
        found = (pos < len(ks)) & (ks[np.minimum(pos, len(ks) - 1)] == q) if len(ks) else np.zeros(len(q), bool)
        self.v[pos[found & ~zero]] = vals[found & ~zero]
        keep = np.ones(len(ks), bool)
        keep[pos[found & zero]] = False
        ins = ~found & ~zero
        self.k, self.v = self.k[keep], self.v[keep]
        if ins.any():
            o = np.argsort(q[ins], kind="stable")
            nk, nv = keys[ins][o], vals[ins][o]
            p = np.searchsorted(self.k.view("S32").ravel(), nk.view("S32").ravel())
            self.k, self.v = np.insert(self.k, p, nk, axis=0), np.insert(self.v, p, nv, axis=0)


def build_state(rng, na, scale):
    """the default shape: account fields (keys, nonces, balances, code hashes), the load's slot arrays and each account's
    storage -> (akeys, nonce, bal, code, slot_acc, skeys, svals, store)"""
    sizes = np.zeros(na, np.int64)
    sizes[0] = int(2_000_000 * scale)
    sizes[1:31] = int(100_000 * scale)
    sizes[31:50_031] = max(1, int(100 * scale))
    akeys, nonce, bal, code = rand_rows(rng, na), rng.integers(0, 1 << 40, na).astype(np.uint64), rand_rows(rng, na), rand_rows(rng, na)
    bal[:, :20] = 0
    ns = int(sizes.sum())
    slot_acc = np.repeat(np.arange(na, dtype=np.uint32), sizes)
    skeys, svals = rand_rows(rng, ns), rand_vals(rng, ns)
    off = np.concatenate([[0], np.cumsum(sizes)])
    store = {a: Storage(skeys[off[a]:off[a + 1]], svals[off[a]:off[a + 1]]) for a in np.nonzero(sizes)[0]}
    return akeys, nonce, bal, code, slot_acc, skeys, svals, store


def make_block(rng, store, small, na, nonce, bal):
    """one block: 30 writes in the 2M account, 1,000 in five 100k accounts, ~14 each in 1,000 small ones; 3,000 accounts
    touched.  Applies it to `store`, `nonce` and `bal` -> (touched, with_slots, slot_index, sk, sv)"""
    plan = [(0, 30)] + [(int(a), 200) for a in rng.choice(np.arange(1, 31), 5, replace=False)]
    plan += [(int(a), 14 if i < 970 else 13) for i, a in enumerate(rng.choice(small, 1000, replace=False))]  # 15,000 in all
    sa, sk, sv = [], [], []
    for a, cnt in plan:
        s = store[a]
        kinds = rng.choice(3, cnt, p=[0.7, 0.2, 0.1])  # update / insert / delete
        n_old = int((kinds != 1).sum())
        pick = rng.choice(len(s.k), min(n_old, len(s.k)), replace=False)
        k = rand_rows(rng, cnt)
        old = np.nonzero(kinds != 1)[0][: len(pick)]
        k[old] = s.k[pick]
        v = rand_vals(rng, cnt)
        v[kinds == 2] = 0
        sa.append(np.full(cnt, a, np.int64)); sk.append(k); sv.append(v)
        s.write(k, v)
    sa, sk, sv = np.concatenate(sa), np.concatenate(sk), np.concatenate(sv)
    with_slots = [a for a, _ in plan]
    others = rng.choice(np.arange(50_031, na), 3000 - len(with_slots), replace=False)
    touched = np.array(with_slots + [int(x) for x in others], np.int64)
    bal[touched, 31] += 1
    nonce[touched] += 1
    index = {int(a): i for i, a in enumerate(touched)}
    slot_index = np.array([index[int(a)] for a in sa], np.uint32)
    return touched, with_slots, slot_index, sk, sv


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every storage size (0.01 for a quick run)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--blocks", type=int, default=20)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    rng = np.random.default_rng(args.seed)
    gpu_name = card()
    na = args.accounts
    akeys, nonce, bal, code, slot_acc, skeys, svals, store = build_state(rng, na, args.scale)
    ns = len(skeys)

    ctx = gpu.Context(0)
    st = ctx.resident_state()
    ctx.reset_stats()
    t0 = time.perf_counter()
    root, sroots = st.apply(akeys, nonce, bal, code, None, slot_acc, skeys, svals, storage_roots=True)
    load_ms = (time.perf_counter() - t0) * 1e3
    load_stats = ctx.stats()
    del slot_acc, skeys, svals
    # kind 1 loaded with the same leaves (storage roots from the resident load; the per-block roots are what is compared)
    trie = ctx.trie_open(0, kind=1)
    leaves = [leaf(nonce[i], bal[i].tobytes(), sroots[i].tobytes(), code[i].tobytes()) for i in range(na)]
    voff = np.concatenate([[0], np.cumsum([len(x) for x in leaves])]).astype(np.uint32)
    assert trie.update(akeys.reshape(-1), np.frombuffer(b"".join(leaves), np.uint8), voff, na) == root, "load roots differ"
    del leaves
    sroot = {a: sroots[a].tobytes() for a in store}

    with_storage = np.array(sorted(store), np.int64)
    small = with_storage[with_storage >= 31]
    legs = {"resident": [], "kind1": []}
    for b in range(args.warmup + args.blocks):
        touched, with_slots, slot_index, sk, sv = make_block(rng, store, small, na, nonce, bal)

        # ---- resident ----
        ctx.reset_stats()
        t0 = time.perf_counter()
        r_root, r_sroots = st.apply(akeys[touched], nonce[touched], bal[touched], code[touched], None, slot_index, sk, sv, storage_roots=True)
        r_ms = (time.perf_counter() - t0) * 1e3
        r_stats = ctx.stats()

        # ---- kind 1: whole storage of every touched account with storage, one batched M call, then the account leaves ----
        parts = [store[a] for a in with_slots]
        kk = np.concatenate([p.k for p in parts]).reshape(-1)
        vv = np.concatenate([np.concatenate([np.full((len(p.v), 1), 0xa0, np.uint8), p.v], axis=1) for p in parts]).reshape(-1)
        nk = sum(len(p.k) for p in parts)
        koff = (np.arange(nk + 1, dtype=np.uint64) * 32).astype(np.uint32)
        vo = np.arange(nk + 1, dtype=np.uint64) * 33
        seg = np.concatenate([[0], np.cumsum([len(p.k) for p in parts])]).astype(np.uint32)
        ctx.reset_stats()
        t0 = time.perf_counter()
        roots = ctx.mpt_roots(kk, koff, vv, vo, seg, len(parts))
        t_m = time.perf_counter()
        for a, rt in zip(with_slots, roots):
            sroot[a] = rt
        lv = [leaf(nonce[a], bal[a].tobytes(), sroot.get(int(a), EMPTY_ROOT), code[a].tobytes()) for a in touched]
        lo = np.concatenate([[0], np.cumsum([len(x) for x in lv])]).astype(np.uint32)
        t_l = time.perf_counter()
        k_root = trie.update(np.ascontiguousarray(akeys[touched]).reshape(-1), np.frombuffer(b"".join(lv), np.uint8), lo, len(touched))
        k_ms = (t_m - t0 + time.perf_counter() - t_l) * 1e3
        k_stats = ctx.stats()
        assert r_root == k_root, f"block {b}: roots differ"
        for i, a in enumerate(with_slots):
            assert r_sroots[i].tobytes() == sroot[a], f"block {b}: storage root of account {a} differs"
        if b >= args.warmup:
            legs["resident"].append((r_ms, r_stats))
            legs["kind1"].append((k_ms, k_stats))

    for name, rows in legs.items():
        ms = np.array([r[0] for r in rows])
        st_ = [r[1] for r in rows]
        print(json.dumps({"leg": name, "gpu": gpu_name, "accounts": na, "slots": ns, "blocks": len(rows),
                          "apply_ms_median": round(float(np.median(ms)), 3), "apply_ms_min": round(float(ms.min()), 3),
                          "apply_ms_max": round(float(ms.max()), 3), "launches": int(np.median([s["launches"] for s in st_])),
                          "h2d_bytes": int(np.median([s["h2d_bytes"] for s in st_])),
                          "keccak_msgs": int(np.median([s["keccak_msgs"] for s in st_])),
                          "load_ms": round(load_ms, 1) if name == "resident" else None,
                          "load_keccak_msgs": load_stats["keccak_msgs"] if name == "resident" else None}))
    print(json.dumps({"roots_agree": True, "device_bytes": st.info()["device_bytes"], "gpu": gpu_name}))
    st.close()
    trie.close()
    ctx.close()


if __name__ == "__main__":
    main()
