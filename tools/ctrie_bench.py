#!/usr/bin/env python3
"""U kind 0 (the resident complete trie): open at depths 6 and 7, and 100k-leaf updates of the depth-6 trie through each
leaf stage -- fused (pinned host memory, 78-byte values), general (the same with one 600-byte value) and device pointers.
Every call is timed up to a device synchronise after warm-up; prints one JSON line with median / min / max in ms and the
launches and Keccak messages per update.  Give it a library path to compare two builds:
  python tools/ctrie_bench.py [path/to/libphantgpu.so] [--steps N]
Needs a GPU.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from phant_b200 import gpu  # noqa: E402

DEPTH, N = 6, 100_000


def summary(seconds):
    ms = sorted(1e3 * x for x in seconds)
    return {"median": ms[len(ms) // 2], "min": ms[0], "max": ms[-1]}


def update_set(rng, big):
    """N distinct leaf positions of the depth-6 trie (its first 3 key bytes), 78-byte values, one of 600 bytes if `big`"""
    pos = rng.choice(16 ** DEPTH, size=N, replace=False).astype(np.uint32)
    keys = rng.integers(0, 256, (N, 32), dtype=np.uint8)
    keys[:, 0], keys[:, 1], keys[:, 2] = (pos >> 16) & 0xff, (pos >> 8) & 0xff, pos & 0xff
    lens = np.full(N, 78)
    if big:
        lens[0] = 600
    voff = np.zeros(N + 1, np.uint32)
    voff[1:] = np.cumsum(lens)
    vals = rng.integers(0, 256, int(voff[-1]), dtype=np.uint8)
    return np.ascontiguousarray(keys.reshape(-1)), vals, voff


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("lib", nargs="?", help="libphantgpu.so to load (default: the tree's own)")
    ap.add_argument("--steps", type=int, default=20, help="timed updates per case")
    ap.add_argument("--open-steps", type=int, default=5, help="timed opens per depth")
    a = ap.parse_args()
    if a.lib:
        gpu.LIB_PATH = os.path.abspath(a.lib)
    import torch

    ctx = gpu.Context(0)
    out = {"lib": gpu.LIB_PATH}
    for depth in (6, 7):
        ctx.trie_open(depth).close()  # warm-up
        ts = []
        for _ in range(a.open_steps):
            t0 = time.perf_counter()
            t = ctx.trie_open(depth)
            ctx.synchronize()
            ts.append(time.perf_counter() - t0)
            t.close()
        out[f"open{depth}_ms"] = summary(ts)

    rng = np.random.default_rng(46)
    t = ctx.trie_open(DEPTH)
    for case in ("fused", "general", "device"):
        sets = [update_set(rng, case == "general") for _ in range(4)]
        if case == "device":
            sets = [[torch.from_numpy(x).cuda() for x in s] for s in sets]
            torch.cuda.synchronize()
            ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
        else:
            sets = [[torch.from_numpy(x).pin_memory() for x in s] for s in sets]
        for s in sets[:2]:
            t.update(*s, N)
        ctx.synchronize()
        ctx.reset_stats()
        ts = []
        for i in range(a.steps):
            s = sets[i % len(sets)]
            t0 = time.perf_counter()
            t.update(*s, N)
            ctx.synchronize()
            ts.append(time.perf_counter() - t0)
        ctx.set_flags(0)
        st = ctx.stats()
        out[f"update_{case}_ms"] = summary(ts)
        out[f"update_{case}_launches"] = st["launches"] / a.steps
        out[f"update_{case}_keccak_msgs"] = st["keccak_msgs"] / a.steps
    t.close()
    ctx.close()
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
