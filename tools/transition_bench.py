"""State transition roots (phant_gpu_transition_roots) on the resident bench's state, block by block and 64 blocks per call.

The state and the blocks are those of tools/resident_state_bench.py: 1,000,000 accounts and about 10M slots; each block
touches 3,000 accounts and writes 15,000 slots.  Every block is a transition from the same pre-state.  Set-up, untimed:
the state is loaded into the resident world state (which also gives every storage root), the oracle builds the pre-state
tries on the host and cuts each block's witness from them (the proofs of the listed keys and of each deleted key's nearest
surviving neighbours, as tests/transition_oracle.py states), and each block's expected root comes from the resident world
state (apply, then revert(1)).  Timed, host wall clock around the synchronous calls:

  1 block/call    one phant_gpu_transition_roots call per block
  64 blocks/call  all blocks in one call (blocks validated against their own parent roots, sharing one node set)

Reported per leg: ms per call and per block, launches, H2D bytes and Keccak messages per call, with the card's name and
power limit read in the same run.  Every root is checked against the resident world state.

    python tools/transition_bench.py [--accounts 1000000] [--scale 1.0] [--blocks 64] [--warmup 2]
"""
import argparse
import bisect
import json
import os
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", "tests"))
import oracle_lib  # noqa: E402
from phant_b200 import gpu  # noqa: E402
from resident_state_bench import build_state, card, leaf, make_block, rlp_bytes  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--accounts", type=int, default=1_000_000)
    ap.add_argument("--scale", type=float, default=1.0, help="multiplies every storage size (0.01 for a quick run)")
    ap.add_argument("--blocks", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--seed", type=int, default=1)
    args = ap.parse_args()
    rng = np.random.default_rng(args.seed)
    gpu_name = card()
    na = args.accounts
    akeys, nonce, bal, code, slot_acc, skeys, svals, store = build_state(rng, na, args.scale)
    ctx = gpu.Context(0)
    st = ctx.resident_state()
    st.set_journal(1)
    pre, sroots = st.apply(akeys, nonce, bal, code, None, slot_acc, skeys, svals, storage_roots=True)
    del slot_acc, skeys, svals
    o = oracle_lib.get()
    # the pre-state on the host: the account trie, and each storage trie as it is first needed
    order = np.argsort(akeys.view("S32").ravel(), kind="stable")
    sorted_keys = [akeys[i].tobytes() for i in order]
    acc_trie = o.trie([(akeys[i].tobytes(), leaf(nonce[i], bal[i].tobytes(), sroots[i].tobytes(), code[i].tobytes())) for i in order])
    pre_store = {a: (s.k.copy(), s.v.copy()) for a, s in store.items()}
    tries = {}

    def storage_trie(a):
        if a not in tries:
            k, v = pre_store[a]
            ks = [x.tobytes() for x in k]
            tries[a] = (o.trie([(kk, rlp_bytes(vv.tobytes())) for kk, vv in zip(ks, v)]), ks)
        return tries[a]

    def prove_with_neighbours(trie, keys, listed, gone, out):
        for k in listed:
            out.update(dict.fromkeys(trie.prove(k)))
            if k not in gone:
                continue
            i = bisect.bisect_left(keys, k)
            for j, step in ((i - 1, -1), (i + (1 if i < len(keys) and keys[i] == k else 0), 1)):
                while 0 <= j < len(keys) and keys[j] in gone:
                    j += step
                if 0 <= j < len(keys):
                    out.update(dict.fromkeys(trie.prove(keys[j])))

    with_storage = np.array(sorted(store), np.int64)
    small = with_storage[with_storage >= 31]
    blocks, want = [], []
    for b in range(args.blocks + args.warmup):
        touched, with_slots, slot_index, sk, sv = make_block(rng, store, small, na, nonce, bal)
        d = dict(account_keys32=akeys[touched], nonce=nonce[touched].copy(), balance32=bal[touched].copy(), code_hash32=code[touched],
                 slot_account=slot_index, slot_keys32=sk, slot_vals32=sv)
        want.append(st.apply(**d))
        st.revert(1)
        nodes = {}
        prove_with_neighbours(acc_trie, sorted_keys, [akeys[a].tobytes() for a in touched], set(), nodes)
        for a in with_slots:
            mine = slot_index == np.where(touched == a)[0][0]
            t, ks = storage_trie(a)
            listed = [x.tobytes() for x in sk[mine]]
            gone = {x.tobytes() for x, v in zip(sk[mine], sv[mine]) if not v.any()}
            prove_with_neighbours(t, ks, listed, gone, nodes)
        blocks.append((list(nodes), d))

    def call(bs):
        nodes = list(dict.fromkeys(n for b in bs for n in b[0]))
        data, off = oracle_lib.csr(nodes, np.uint64)
        cat = {k: np.concatenate([b[1][k] for b in bs]) for k in bs[0][1] if k != "slot_account"}
        base = np.cumsum([0] + [len(b[1]["nonce"]) for b in bs])[:-1]
        sa = np.concatenate([b[1]["slot_account"] + np.uint32(base[i]) for i, b in enumerate(bs)]).astype(np.uint32)
        ab = np.concatenate([np.full(len(b[1]["nonce"]), i, np.uint32) for i, b in enumerate(bs)])
        pres = np.frombuffer(pre * len(bs), np.uint8)
        ctx.synchronize()
        ctx.reset_stats()
        t0 = time.perf_counter()
        roots, status = ctx.transition_roots(data, off, pres, account_block=ab, slot_account=sa, **cat)
        ms = (time.perf_counter() - t0) * 1e3
        return roots, status, ms, ctx.stats()

    warm, timed = blocks[: args.warmup], blocks[args.warmup:]
    for b in warm:
        call([b])
    ms1, stats1 = [], []
    for i, b in enumerate(timed):
        roots, status, ms, s = call([b])
        assert status[0] == 1 and roots[0].tobytes() == want[args.warmup + i], i
        ms1.append(ms)
        stats1.append(s)
    call(timed)  # the shape of the many-block call, warmed
    roots, status, ms_many, s_many = call(timed)
    assert list(status) == [1] * len(timed) and [r.tobytes() for r in roots] == want[args.warmup:]
    med = lambda xs: float(np.median(xs))  # noqa: E731
    print(json.dumps({"leg": "1 block/call", "gpu": gpu_name, "accounts": na, "blocks": len(timed), "ms_per_call_median": round(med(ms1), 2),
                      "launches": med([s["launches"] for s in stats1]), "h2d_bytes": med([s["h2d_bytes"] for s in stats1]),
                      "keccak_msgs": med([s["keccak_msgs"] for s in stats1])}))
    print(json.dumps({"leg": f"{len(timed)} blocks/call", "gpu": gpu_name, "accounts": na, "ms_per_call": round(ms_many, 2),
                      "ms_per_block": round(ms_many / len(timed), 3), "launches": s_many["launches"], "h2d_bytes": s_many["h2d_bytes"],
                      "keccak_msgs": s_many["keccak_msgs"]}))
    print(json.dumps({"roots_agree": True, "gpu": gpu_name}))
    st.close()


if __name__ == "__main__":
    main()
