"""What an account or storage range of the resident world state (phant_gpu_resident_state_range) returns, stated on the
Python model, and the request shapes the range tests ask with."""
ZERO_KEY, MAX_KEY = bytes(32), b"\xff" * 32


def add(k, d):
    """the 32-byte key k + d, clamped to [0, 2^256 - 1]"""
    return min(max(int.from_bytes(k, "big") + d, 0), (1 << 256) - 1).to_bytes(32, "big")


def expect(keys, origin, limit, max_entries):
    """keys: the keys present at the root, sorted.  (the keys the range returns, more)"""
    inside = [k for k in keys if origin <= k <= limit]
    return inside[:max_entries], len(inside) > max_entries


def bounds(keys):
    """origins and limits around a key set: the ends of the key space, each key, and its neighbours"""
    out = {ZERO_KEY, MAX_KEY}
    for k in keys:
        out.update((k, add(k, 1), add(k, -1)))
    return sorted(out)


def ranges_over(keys, rng, n, maxes=(0, 1, 2, 3, 10, (1 << 32) - 1)):
    """n (origin, limit, max) triples: origins and limits drawn from bounds(keys) (origin > limit included), the full range
    with every max"""
    b = bounds(keys)
    out = [(ZERO_KEY, MAX_KEY, m) for m in maxes]
    for _ in range(n):
        o, l = b[int(rng.integers(0, len(b)))], b[int(rng.integers(0, len(b)))]
        out.append((o, l, int(maxes[int(rng.integers(0, len(maxes)))])))
    return out
