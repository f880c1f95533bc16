#!/usr/bin/env python3
"""Pre-state reads (entry point P) on the C5 shape: synth_blocks' node arena as one node set, per transaction the sender A and
contract B under the block's state root (n_roots = n_accounts) and B's two slots -- 600k account reads and 600k slot reads
at 1000 blocks x 300 tx.  Device pointers.  Times, alternating in one process after warm-up:
  P:        one phant_gpu_read_state call, timed with CUDA events on the context's stream (and, for comparison with the
            two-step path, host wall clock around the synchronised call);
  two-step: what a caller does without P -- W over the accounts, the storage roots decoded on the host from the proven
            account bodies (the caller holds the witness bytes there), W over the slots under those roots.  Host wall clock:
            the middle step runs on the host, which device events do not see.  The host decode here is a PYTHON loop over
            host.py's strict RLP decoder: its time says what a Python caller pays, not what a native caller would.
Development tool: prints the card, its power limit and one JSON line.
  python tools/state_read_bench.py --blocks 1000 --txs 300 --steps 3
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def power_limit_w():
    """the board power limit as the driver reports it (read-only query), or None"""
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30)
        return float(r.stdout.strip().splitlines()[0])
    except (OSError, ValueError, IndexError, subprocess.SubprocessError):
        return None


def storage_root(body):
    """the third item of a proven account body rlp([nonce, balance, storageRoot, codeHash]) (host.py's strict RLP decoder),
    or None"""
    from phant_b200.host import InvalidWitness, _rlp_header, _rlp_list_items
    try:
        is_list, ps, pe = _rlp_header(body, 0, len(body))
        items = _rlp_list_items(body, ps, pe) if is_list and pe == len(body) else []
    except InvalidWitness:
        return None
    if len(items) != 4 or any(it[0] for it in items) or items[2][3] - items[2][2] != 32:
        return None
    return body[items[2][2]:items[2][3]]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=1000)
    ap.add_argument("--txs", type=int, default=300)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    from phant_b200 import gpu, synth_blocks
    dev = torch.device("cuda", 0)
    ctx = gpu.Context(0)
    w = synth_blocks.synth_blocks(ctx, dev, 0, a.blocks, txs=a.txs)
    n_tx = w["n_proofs"] // 4
    keys, roots = w["keys32"].view(n_tx, 4, 32), w["roots32"].view(n_tx, 4, 32)
    akeys, aroots = keys[:, :2].reshape(-1).contiguous(), roots[:, :2].reshape(-1).contiguous()
    skeys = keys[:, 2:].reshape(-1).contiguous()
    na = ns = 2 * n_tx
    slot_acc = 2 * torch.arange(ns, device=dev).div(2, rounding_mode="floor") + 1
    sacc = slot_acc.to(torch.int32)
    nodes_host = w["nodes"].cpu().numpy()  # a caller decoding on the host holds the witness bytes there
    u8 = lambda n: torch.zeros(n, dtype=torch.uint8, device=dev)
    out = dict(account_status=u8(na), nonce=torch.zeros(na, dtype=torch.int64, device=dev), balance32=u8(32 * na), storage_root32=u8(32 * na),
               code_hash32=u8(32 * na), code_index=torch.zeros(na, dtype=torch.int32, device=dev), slot_status=u8(ns), slot_vals32=u8(32 * ns))
    a_st, a_vo, a_vl = u8(na), torch.zeros(na, dtype=torch.int64, device=dev), torch.zeros(na, dtype=torch.int32, device=dev)
    s_st, s_vo, s_vl = u8(ns), torch.zeros(ns, dtype=torch.int64, device=dev), torch.zeros(ns, dtype=torch.int32, device=dev)
    torch.cuda.synchronize()
    ctx.set_flags(gpu.FLAG_DEVICE_PTRS)

    side = torch.cuda.Stream(device=dev)  # the library and the events share one stream
    ctx.set_stream(side.cuda_stream)

    def run_p():
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        e0.record(side)
        ctx.read_state(w["n_nodes"], w["nodes"], w["node_off"], na, akeys, aroots, na, ns, skeys, sacc, nodes_bytes=w["n_bytes"], **out)
        e1.record(side)
        ctx.synchronize()
        wall = time.perf_counter() - t0
        return e0.elapsed_time(e1) * 1e-3, wall

    def run_two_step():
        t0 = time.perf_counter()
        ctx.verify_witness(w["n_nodes"], w["nodes"], w["node_off"], na, akeys, aroots, na, None, a_st, a_vo, a_vl, nodes_bytes=w["n_bytes"])
        ctx.synchronize()
        t1 = time.perf_counter()
        st, vo, vl = a_st.cpu().numpy(), a_vo.cpu().numpy(), a_vl.cpu().numpy()
        sroots = np.zeros((na, 32), np.uint8)
        for i in np.nonzero(st == 1)[0]:
            r = storage_root(nodes_host[vo[i]:vo[i] + vl[i]].tobytes())
            if r is not None:
                sroots[i] = np.frombuffer(r, np.uint8)
        d_sroots = torch.from_numpy(sroots[slot_acc.cpu().numpy()].reshape(-1)).to(dev)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        ctx.verify_witness(w["n_nodes"], w["nodes"], w["node_off"], ns, skeys, d_sroots, ns, None, s_st, s_vo, s_vl, nodes_bytes=w["n_bytes"])
        ctx.synchronize()
        t3 = time.perf_counter()
        return t3 - t0, (t1 - t0, t2 - t1, t3 - t2)

    for _ in range(a.warmup):
        run_p()
        run_two_step()
    p_s, p_wall, two_s, parts = [], [], [], []
    ctx.reset_stats()
    for _ in range(a.steps):
        ev_s, wall_s = run_p()
        p_s.append(ev_s)
        p_wall.append(wall_s)
        t, pt = run_two_step()
        two_s.append(t)
        parts.append(pt)
    st = ctx.stats()
    ctx.set_flags(0)
    ctx.set_stream(None)
    ok = bool((out["slot_status"] == s_st).all()) and bool((out["account_status"] == a_st).all())
    pm = np.median(parts, axis=0)
    print(json.dumps({"config": f"P: {a.blocks} blocks x {a.txs} tx (C5 shape), {na} account reads + {ns} slot reads, device pointers",
                      "gpu": torch.cuda.get_device_name(0), "power_limit_w": power_limit_w(), "unique_nodes": w["n_nodes"],
                      "node_bytes": w["n_bytes"], "p_ms_median_cuda_events": 1e3 * float(np.median(p_s)), "p_ms_all_cuda_events": [1e3 * x for x in p_s],
                      "p_ms_median_wall": 1e3 * float(np.median(p_wall)),
                      "two_step_ms_median_wall": 1e3 * float(np.median(two_s)),
                      "two_step_parts_ms": {"w_accounts": 1e3 * pm[0], "host_decode_python_loop": 1e3 * pm[1], "w_slots": 1e3 * pm[2]},
                      "walk_kernel_ms_per_step_p_and_w": st["walk_ms"] / a.steps, "statuses_agree": ok,
                      "accounts_present": int((out["account_status"] == 1).sum()), "slots_present": int((out["slot_status"] == 1).sum())}))
    ctx.close()


if __name__ == "__main__":
    main()
