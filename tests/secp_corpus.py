"""Adversarial operands for the arithmetic of phant_b200/csrc/secp256k1.cuh, the Python values they must produce, and a
model of which path each case takes through the code.

Operands are built by limb pattern (every 64-bit limb one of 0, 1, 2^32 - 1, 2^32, 2^63, 2^64 - 2, 2^64 - 1 or random, so
that runs of all-ones limbs carry through every column), from boundary values, from pairs whose sum or difference lands on
a boundary, and -- for fp_reduce and sc_mul -- from 512-bit values built to take the rare folds: fp_reduce's second wrap
(k = 1), its folded value in [p, 2^256), and sc_mul's third and fourth fold rounds.  Uniform random operands almost never
reach those.  Everything is seeded: the same cases every run.

check(run, op) runs one op's cases through `run(op_code, inputs) -> outputs` (the device build, tests/devcheck/
secp_device.cu, or the host build, tests/hostcheck/ecrecover_host.cpp; both wrap tests/devcheck/secp_ops.cuh) and asserts
every output word.  path_counts(op) says how many cases take each tracked path; the tests hold those counts above floors so
that an edit cannot quietly drop a corner."""
import functools
from collections import Counter

import numpy as np

import secp_ref as ref
from secp_ref import C, K, N, P

M256 = 2 ** 256
IN_WORDS, OUT_WORDS = 20, 13
OPS = ["add_raw", "sub_raw", "mul_wide", "fp_reduce", "fp_add", "fp_sub", "fp_neg", "fp_mul", "fp_inv", "fp_sqrt_candidate",
       "sc_mul", "sc_neg", "sc_inv", "jac_double", "jac_add_affine", "to_affine", "ecrecover"]
CODE = {op: i for i, op in enumerate(OPS)}

# cases per op: the limb-level ops are cheap everywhere; inverses, square roots and points cost a few hundred
# multiplications each on the device side and a pow() or an inversion each on the Python side
LIMB_CASES = 200_000
SLOW_CASES = 20_000
POINT_CASES = 20_000
RECOVER_CASES = 600
SIZES = {op: LIMB_CASES for op in OPS}
SIZES.update(fp_inv=SLOW_CASES, fp_sqrt_candidate=SLOW_CASES, sc_inv=SLOW_CASES, jac_double=POINT_CASES,
             jac_add_affine=POINT_CASES, to_affine=POINT_CASES, ecrecover=RECOVER_CASES)

LIMB_PATTERNS = np.array([0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 63, 2 ** 64 - 2, 2 ** 64 - 1], np.uint64)
BOUNDARY = [0, 1, 2, P - 1, P - 2, P - C, C, C - 1, (P + 1) // 2, N - 1, N, N + 1, M256 - 1, M256 - 2, M256 - 2 ** 64, P, P + 1,
            2 ** 255, 2 ** 128 - 1, 2 ** 192 - 1, K, M256 - C - 1]
SUM_TARGETS = [P - 1, P, P + 1, M256 - 1, M256, M256 + C - 1]
DIFF_TARGETS = [-1, 0, 1, P - 1, P, -(P - 1), -C, C]


# ---- operands ----
def patterned(rng, count, limbs=4):
    """count integers of `limbs` 64-bit limbs, each limb a pattern value or (one time in eight) random"""
    idx = rng.integers(0, len(LIMB_PATTERNS) + 1, size=(count, limbs))
    rnd = np.frombuffer(rng.bytes(8 * count * limbs), np.uint64).reshape(count, limbs)
    w = np.where(idx == len(LIMB_PATTERNS), rnd, LIMB_PATTERNS[np.minimum(idx, len(LIMB_PATTERNS) - 1)]).tobytes()
    s = 8 * limbs
    return [int.from_bytes(w[i * s:(i + 1) * s], "little") for i in range(count)]


def operands(rng, count, bound=M256):
    """count integers in [0, bound): half by limb pattern, the rest boundary values +- a few, uniform and small values"""
    pat = patterned(rng, count)
    kind = rng.integers(0, 8, size=count)
    delta = rng.integers(-3, 4, size=count)
    pick = rng.integers(0, len(BOUNDARY), size=count)
    out = []
    for i in range(count):
        k = int(kind[i])
        if k < 4:
            v = pat[i]
        elif k < 6:
            v = (BOUNDARY[pick[i]] + int(delta[i])) % M256
        elif k == 6:
            v = int.from_bytes(rng.bytes(32), "little")
        else:
            v = int.from_bytes(rng.bytes(int(rng.integers(1, 9))), "little")
        out.append(v if v < bound else v % bound)
    return out


def pair_with(a, target, bound, diff=False):
    """(a', b) with a' + b == target (or a' - b == target), both in [0, bound), a' derived from a; None when impossible"""
    lo, hi = (max(0, target), min(bound - 1, bound - 1 + target)) if diff else (max(0, target - bound + 1), min(bound - 1, target))
    if lo > hi:
        return None
    a = lo + a % (hi - lo + 1)
    return a, (a - target if diff else target - a)


def pairs(rng, count, bound):
    """operand pairs in [0, bound): a quarter of them sum or subtract to a boundary, the rest independent"""
    xs, ys = operands(rng, count, bound), operands(rng, count, bound)
    kind = rng.integers(0, 8, size=count)
    tgt = rng.integers(0, 64, size=count)
    out = []
    for i in range(count):
        a, b = xs[i], ys[i]
        if kind[i] == 0:
            a, b = pair_with(a, SUM_TARGETS[tgt[i] % len(SUM_TARGETS)], bound) or (a, b)
        elif kind[i] == 1:
            a, b = pair_with(a, DIFF_TARGETS[tgt[i] % len(DIFF_TARGETS)], bound, diff=True) or (a, b)
        out.append((a, b))
    return out


def reduce_inputs(rng, count):
    """512-bit T for fp_reduce: a quarter limb patterns, a quarter products, half built for the rare paths (see below)"""
    out = patterned(rng, count // 4, limbs=8)
    out += [a * b for a, b in pairs(rng, count // 4, M256)]
    his = patterned(rng, count - len(out))
    for i, hi in enumerate(his):
        # T = lo + hi 2^256 folds to r = lo + hi C = L + q 2^256 with q = floor(hi C / 2^256) when L >= (hi C mod 2^256);
        # the second fold then adds q C to L: L >= 2^256 - q C wraps (k = 1), L + q C in [p, 2^256) needs fp_norm
        q = hi * C >> 256
        j = int.from_bytes(rng.bytes(8), "little")
        if i % 8 == 7:                                          # limb 4 at its maximum, C: hi = 2^256 - 1 - e, lo >= (e + 1) C
            out.append(M256 - 1 - j % 2 ** 40 + ((M256 - 1 - j % 3) << 256))
            continue
        L = M256 - 1 - j % (q * C) if i % 2 == 0 and q else P - q * C + j % C   # k = 1, or the folded value in [p, 2^256)
        out.append((L - hi * C) % M256 + (hi << 256))
    out += [M256 * M256 - 1, (M256 - 1) * M256, M256 - 1, P, P * P, (P - 1) * (P - 1), (M256 - 1) ** 2]
    return out


def sc_pairs(rng, count):
    """sc_mul operands: independent pairs (one, two or three fold rounds) and a * b = c (mod n) with c just above
    K = 2^256 - n, whose folding can end on c + n >= 2^256 and so take a fourth round"""
    out = pairs(rng, count // 2, M256)
    for _ in range(count - len(out)):
        a = int.from_bytes(rng.bytes(32), "little") % (N - 1) + 1
        c = K + int.from_bytes(rng.bytes(17), "little") % (7 * K)
        out.append((a, c * ref.sc_inv(a) % N))
    return out


def points(rng, count):
    """count affine curve points: random multiples of G walked forward by a random step, plus G and -G"""
    pts = [ref.G, ref.neg(ref.G)]
    step = ref.mul(int.from_bytes(rng.bytes(32), "little") % N, ref.G)
    cur = ref.mul(int.from_bytes(rng.bytes(32), "little") % N, ref.G)
    while len(pts) < count:
        if len(pts) % 500 == 0:
            cur = ref.mul(int.from_bytes(rng.bytes(32), "little") % N, ref.G)
        cur = ref.add(cur, step)
        pts.append(cur)
    return pts


def jacobian(rng, pt, kind):
    """pt as (X, Y, Z) = (x z^2, y z^3, z), z random (kind 0), 1 (kind 1), p - 1 (kind 2); infinity has Z = 0"""
    if pt is ref.INF:
        return (0, 1, 0) if kind else (int.from_bytes(rng.bytes(32), "little") % P, int.from_bytes(rng.bytes(32), "little") % P, 0)
    z = [int.from_bytes(rng.bytes(32), "little") % (P - 1) + 1, 1, P - 1][kind]
    return (pt[0] * z * z % P, pt[1] * z ** 3 % P, z)


def affine_of(X, Y, Z):
    if Z == 0:
        return ref.INF
    zi = ref.fp_inv(Z)
    return (X * zi * zi % P, Y * zi ** 3 % P)


# ---- the cases of one op: tuples of ints, laid out in words by IN_LAYOUT ----
@functools.lru_cache(maxsize=None)
def cases(op):
    rng = np.random.default_rng(1000 + CODE[op])
    n = SIZES[op]
    if op in ("add_raw", "sub_raw", "mul_wide"):
        return pairs(rng, n, M256)
    if op == "fp_reduce":
        return [(t,) for t in reduce_inputs(rng, n)]
    if op in ("fp_add", "fp_sub"):
        return pairs(rng, n, P)
    if op == "fp_mul":
        return pairs(rng, n // 2, P) + pairs(rng, n - n // 2, M256)   # fp_reduce folds any 512-bit product
    if op == "sc_mul":
        return sc_pairs(rng, n)
    if op in ("fp_neg", "fp_inv", "fp_sqrt_candidate"):
        return [(a,) for a in operands(rng, n, P)]
    if op in ("sc_neg", "sc_inv"):
        return [(a,) for a in operands(rng, n, N)]
    if op == "ecrecover":
        return recover_cases(rng, n)
    pts = points(rng, 2000)
    pick = rng.integers(0, len(pts), size=(n, 2))
    kind = rng.integers(0, 8, size=(n, 2))
    out = []
    for i in range(n):
        p, q = pts[pick[i, 0]], pts[pick[i, 1]]
        k = int(kind[i, 0])
        if op == "jac_add_affine":
            if k == 1:
                q = p                                  # the same point: the doubling branch
            elif k == 2:
                q = ref.neg(p)                         # opposite points: infinity
            elif k == 3:
                p = ref.INF                            # accumulator at infinity
        elif k == 3:
            p = ref.INF
        zkind = [0, 0, 0, 0, 0, 1, 2, 0][kind[i, 1]] if p is not ref.INF else int(kind[i, 1]) % 2
        out.append(jacobian(rng, p, zkind) + ((q[0], q[1]) if op == "jac_add_affine" else ()))
    return out


def recover_cases(rng, n):
    """(z, r, s, recid): valid signatures from random keys (both parities, high and low s), x = r + n lifts, and random
    tuples with boundary r and s"""
    out = []
    for i in range(n):
        z = int.from_bytes(rng.bytes(32), "little")
        kind = i % 4
        if kind == 0:
            d, k = (int.from_bytes(rng.bytes(32), "little") % (N - 1) + 1 for _ in range(2))
            r, s, recid = ref.sign(d, z, k)
            if i % 8 == 4:
                s, recid = N - s, recid ^ 1             # the other half of s recovers the same key
            out.append((z, r, s, recid))
        elif kind == 1:
            out.append((z, int.from_bytes(rng.bytes(16), "little"), int.from_bytes(rng.bytes(32), "little") % N, 2 + i // 4 % 2))
        elif kind == 2:
            r = [0, 1, N - 1, N, P - N - 1, P - N, P - N + 1, M256 - 1, ref.GX][i // 4 % 9]
            s = [0, 1, N - 1, N, M256 - 1, 7][i // 36 % 6]
            out.append((z, r, s, i // 8 % 4))
        else:
            out.append((z, int.from_bytes(rng.bytes(32), "little"), int.from_bytes(rng.bytes(32), "little"),
                        int(rng.integers(0, 4)) if i % 16 != 3 else int(rng.integers(4, 256))))
    return out


# ---- the Python values ----
def expected(op, case):
    """the exact outputs of one case, as the ints of the output layout (points are compared separately: see check)"""
    a = case[0]
    b = case[1] if len(case) > 1 else None
    if op == "add_raw":
        return [(a + b) % M256, (a + b) >> 256]
    if op == "sub_raw":
        return [(a - b) % M256, 1 if a < b else 0]
    if op == "mul_wide":
        return [a * b]
    if op == "fp_reduce":
        return [a % P]
    if op == "fp_add":
        return [(a + b) % P]
    if op == "fp_sub":
        return [(a - b) % P]
    if op == "fp_neg":
        return [-a % P]
    if op == "fp_mul":
        return [a * b % P]
    if op == "fp_inv":
        return [pow(a, -1, P) if a else 0]          # a^(p-2): 0 for a = 0
    if op == "fp_sqrt_candidate":
        return [pow(a, (P + 1) // 4, P)]
    if op == "sc_mul":
        return [a * b % N]
    if op == "sc_neg":
        return [-a % N]
    if op == "sc_inv":
        return [pow(a, -1, N) if a else 0]          # a^(n-2): 0 for a = 0
    if op == "to_affine":
        q = affine_of(*case)
        return [0, 0, 1] if q is ref.INF else [q[0], q[1], 0]
    if op == "ecrecover":
        return _recovered(case)
    raise KeyError(op)


@functools.lru_cache(maxsize=None)
def _recovered(case):
    z, r, s, recid = case
    pub = ref.recover(z.to_bytes(32, "big"), ref.sig65(r, s, recid))
    return [0, 0, 0] if pub is None else [int.from_bytes(pub[1:33], "big"), int.from_bytes(pub[33:], "big"), 1]


IN_LAYOUT = {"add_raw": [4, 4], "sub_raw": [4, 4], "mul_wide": [4, 4], "fp_reduce": [8], "fp_add": [4, 4], "fp_sub": [4, 4],
             "fp_neg": [4], "fp_mul": [4, 4], "fp_inv": [4], "fp_sqrt_candidate": [4], "sc_mul": [4, 4], "sc_neg": [4],
             "sc_inv": [4], "jac_double": [4, 4, 4], "jac_add_affine": [4, 4, 4, 4, 4], "to_affine": [4, 4, 4],
             "ecrecover": [4, 4, 4, 1]}
OUT_LAYOUT = {"add_raw": [4, 1], "sub_raw": [4, 1], "mul_wide": [8], "fp_reduce": [4], "to_affine": [4, 4, 1],
              "jac_double": [4, 4, 4], "jac_add_affine": [4, 4, 4], "ecrecover": [4, 4, 1]}


def pack(values, layout, width):
    """rows of ints -> (rows, width) uint64, each int in its layout's number of little-endian words"""
    pad = bytes(8 * (width - sum(layout)))
    blob = b"".join(b"".join(v.to_bytes(8 * w, "little") for v, w in zip(row, layout)) + pad for row in values)
    return np.frombuffer(blob, np.uint64).reshape(len(values), width)


def unpack(words, layout):
    """(rows, >= sum(layout)) uint64 -> rows of ints"""
    blob, width = np.ascontiguousarray(words[:, :sum(layout)]).tobytes(), 8 * sum(layout)
    out = []
    for i in range(words.shape[0]):
        row, o = [], i * width
        for w in layout:
            row.append(int.from_bytes(blob[o:o + 8 * w], "little"))
            o += 8 * w
        out.append(row)
    return out


def check(run, op):
    """run every case of `op` through run(op_code, inputs (n, IN_WORDS) uint64) -> outputs (n, OUT_WORDS) uint64 and
    assert each output against Python: exact values, canonical (below p or n), carry words 0 or 1, no unwritten word.
    Returns the number of cases."""
    cs = cases(op)
    inp = pack(cs, IN_LAYOUT[op], IN_WORDS)
    out = run(CODE[op], inp)
    assert out.shape == (len(cs), OUT_WORDS)
    layout = OUT_LAYOUT.get(op, [4])
    if op in ("jac_double", "jac_add_affine"):
        got = unpack(out, layout)
        for case, (X, Y, Z) in zip(cs, got):
            assert X < P and Y < P and Z < P, (op, case, (X, Y, Z))
            p = affine_of(*case[:3])
            want = ref.double(p) if op == "jac_double" else ref.add(p, (case[3], case[4]))
            assert affine_of(X, Y, Z) == want, (op, case, (X, Y, Z))
        return len(cs)
    want = pack([expected(op, c) for c in cs], layout, sum(layout))
    bad = np.nonzero((out[:, :sum(layout)] != want).any(axis=1))[0]
    assert not len(bad), (op, f"{len(bad)} of {len(cs)} cases wrong; first: in", cs[bad[0]], "got", unpack(out[bad[:1]], layout),
                          "want", unpack(want[bad[:1]], layout))
    return len(cs)


# ---- which path each case takes ----
def fp_reduce_paths(t):
    """the fold of fp_reduce as the code does it: lo + hi C (limb 4 = r4), then r4 C into the low four limbs (carry k),
    then k C, then fp_norm when the value is in [p, 2^256)"""
    lo, hi = t % M256, t >> 256
    r = lo + hi * C
    r4 = r >> 256
    o = r % M256 + r4 * C
    k = o >> 256
    o = o % M256 + k * C
    paths = []
    if k:
        paths.append("fp_reduce k = 1")
    if r4 == C:
        paths.append("fp_reduce limb 4 at its maximum")
    if o >= P:
        paths.append("fp_reduce folded value in [p, 2^256)")
    return paths


def carry_paths(name, a, b, sub):
    """carry (borrow) out of every limb: the chain rippled through all four"""
    c, outs = 0, []
    for i in range(4):
        x, y = (a >> 64 * i) & (2 ** 64 - 1), (b >> 64 * i) & (2 ** 64 - 1)
        v = x - y - c if sub else x + y + c
        c = 1 if (v < 0 if sub else v >> 64) else 0
        outs.append(c)
    paths = [f"{name} carry out"] if outs[3] else []
    if all(outs):
        paths.append(f"{name} carry through all four limbs")
    return paths


def path_counts(op):
    counts = Counter()
    for case in cases(op):
        if op in ("add_raw", "sub_raw"):
            counts.update(carry_paths(op, case[0], case[1], op == "sub_raw"))
        elif op == "fp_reduce":
            counts.update(fp_reduce_paths(case[0]))
        elif op == "fp_mul":
            counts.update(fp_reduce_paths(case[0] * case[1]))
        elif op == "fp_add":
            s = case[0] + case[1]
            if s >= M256:
                counts["fp_add carry"] += 1
            elif s >= P:
                counts["fp_add sum in [p, 2^256)"] += 1
        elif op == "fp_sub":
            if case[0] < case[1]:
                counts["fp_sub borrow"] += 1
        elif op == "sc_mul":
            t, rounds = case[0] * case[1], 0
            while t >> 256:
                t, rounds = t % M256 + (t >> 256) * K, rounds + 1
            counts[f"sc_mul fold rounds = {rounds}"] += 1
            if t >= N:
                counts["sc_mul final subtraction of n"] += 1
        elif op == "jac_add_affine":
            p, q = affine_of(*case[:3]), (case[3], case[4])
            counts["jac_add_affine " + ("accumulator at infinity" if p is ref.INF else "same point" if p == q else
                                        "opposite points" if p == ref.neg(q) else "distinct points")] += 1
        elif op in ("jac_double", "to_affine"):
            counts[f"{op} " + ("infinity" if case[2] == 0 else "z = 1" if case[2] == 1 else "z != 1")] += 1
        elif op == "ecrecover":
            counts["ecrecover recovers" if expected(op, case)[2] else "ecrecover rejects"] += 1
    return counts


# floors the corpus must keep: every path of the fold and carry logic taken by this many cases at least
PATH_FLOORS = {
    "add_raw": {"add_raw carry out": 20_000, "add_raw carry through all four limbs": 5_000},
    "sub_raw": {"sub_raw carry out": 20_000, "sub_raw carry through all four limbs": 5_000},
    "fp_reduce": {"fp_reduce k = 1": 10_000, "fp_reduce limb 4 at its maximum": 10, "fp_reduce folded value in [p, 2^256)": 10_000},
    "fp_mul": {"fp_reduce k = 1": 100, "fp_reduce limb 4 at its maximum": 1_000, "fp_reduce folded value in [p, 2^256)": 1_000},
    "fp_add": {"fp_add carry": 5_000, "fp_add sum in [p, 2^256)": 1_000},
    "fp_sub": {"fp_sub borrow": 20_000},
    "sc_mul": {"sc_mul fold rounds = 3": 20_000, "sc_mul fold rounds = 4": 1_000, "sc_mul final subtraction of n": 1_000},
    "jac_add_affine": {"jac_add_affine accumulator at infinity": 1_000, "jac_add_affine same point": 1_000,
                       "jac_add_affine opposite points": 1_000, "jac_add_affine distinct points": 5_000},
    "jac_double": {"jac_double infinity": 1_000, "jac_double z = 1": 1_000, "jac_double z != 1": 5_000},
    "to_affine": {"to_affine infinity": 1_000, "to_affine z = 1": 1_000, "to_affine z != 1": 5_000},
    "ecrecover": {"ecrecover recovers": 150, "ecrecover rejects": 150},
}


# ---- whole signatures for the recovery kernel: every case says what must come out ----
AGREE = "agree"   # no independent statement of the key: the kernel, secp_ref and the oracle must agree


def crafted_signatures():
    """[(label, hash32, sig65, want)]: want is the 65-byte key the case must recover, None when it must be rejected, or
    AGREE.  Valid signatures from known keys (the key is d G: a fact, not an agreement); the double multiplication's
    corners driven on purpose through (u1, u2); the x = r + n lift at its limits; every r / s boundary; recid > 3."""
    rng = np.random.default_rng(77)
    rand = lambda: int.from_bytes(rng.bytes(32), "little") % (N - 1) + 1   # noqa: E731
    out = []

    def add(label, z, r, s, recid, want):
        out.append((label, (z % M256).to_bytes(32, "big"), ref.sig65(r, s, recid), want))

    # valid signatures from known keys: both halves of s (so both parities), hashes at and above n (z >= n is reduced)
    for d in [1, 2, 3, N - 1, N - 2, 2 ** 128, 2 ** 255, rand(), rand()]:
        pub = ref.pubkey(d)
        for k in [1, N - 1, rand()]:
            for z in [0, 1, N - 1, N, N + 1, M256 - 1, int.from_bytes(rng.bytes(32), "little")]:
                try:
                    r, s, recid = ref.sign(d, z, k)
                except ValueError:
                    continue
                add(f"key d={d:#x} k={k:#x} z={z:#x}", z, r, s, recid, pub)
                add(f"key d={d:#x} k={k:#x} z={z:#x} other half of s", z, r, N - s, recid ^ 1, pub)

    # the double multiplication Q = u1 G + u2 R, R = k G, driven through z = -u1 r and s = u2 r (mod n): Q = (u1 + u2 k) G
    def corner(label, k, u1, u2):
        R = ref.mul(k, ref.G)
        r, recid = R[0] % N, (R[1] & 1) | (2 if R[0] >= N else 0)
        z, s = -u1 * r % N, u2 * r % N
        e = (u1 + u2 * k) % N
        want = None if e == 0 else ref.pubkey(e)
        add(f"corner {label}", z, r, s, recid, want)
        if z + N < M256:
            add(f"corner {label}, hash + n", z + N, r, s, recid, want)

    ka = rand()
    for u1, u2 in [(rand(), rand()), (0, rand()), (rand(), 1), (1, 1), (N - 1, N - 1), (0, 1)]:
        corner(f"R = G u1={u1:#x} u2={u2:#x}", 1, u1, u2)                 # G + R through the doubling branch
        corner(f"R = -G u1={u1:#x} u2={u2:#x}", N - 1, u1, u2)            # G + R at infinity: the sel == 3 entry skipped
        corner(f"R = {ka:#x} G u1={u1:#x} u2={u2:#x}", ka, u1, u2)
    corner("acc meets the point it adds", 2, 2, 1)
    corner("acc meets its negation at the last bit", N - 2, 2, 1)        # Q at infinity
    corner("acc meets its negation mid-way", N - 2, 5, 2)
    corner("u1 = n - 1, u2 = 1", 3, N - 1, 1)
    for bits in (1, 2, 8, 64, 128):                                       # long runs of leading zero bits
        for k in (1, 2, N - 1, ka):
            corner(f"short scalars {bits} bits k={k:#x}", k, int(rng.integers(0, 2 ** min(bits, 62))) + (1 << (bits - 1)),
                   int(rng.integers(1, 2 ** min(bits, 62))) | (1 << (bits - 1)))
    for k in (1, 2, 3, N - 1, N - 2, ka):                                # u1 + u2 k = 0: Q at infinity
        u2 = rand()
        corner(f"Q at infinity k={k:#x}", k, -u2 * k % N, u2)

    # the x = r + n lift (recid 2 and 3) at its limits
    for r in [P - N - 1, P - N, P - N + 1, K - 1, K, K + 1]:                 # x = p - 1, p, p + 1 / x = 2^256 - 1, 2^256 (carry out)
        for recid in (2, 3):
            add(f"lift r={r:#x}", int.from_bytes(rng.bytes(32), "little"), r, rand(), recid, AGREE if r + N < P else None)
    lifts = {True: 0, False: 0}
    while min(lifts.values()) < 6:                                       # small r: r + n on the curve or not
        r = int.from_bytes(rng.bytes(int(rng.integers(1, 17))), "little") or 1
        on = ref.lift_x(r + N, 0) is not None
        if lifts[on] < 6:
            lifts[on] += 1
            add(f"lift small r={r:#x} on curve={on}", int.from_bytes(rng.bytes(32), "little"), r, rand(), 2 + lifts[on] % 2,
                AGREE if on else None)

    # every r / s boundary with every recid; recid 4..255 on a signature that is otherwise valid
    for r in [0, 1, N - 1, N, M256 - 1]:
        for s in [0, 1, N - 1, N, M256 - 1]:
            for recid in range(4):
                add(f"bounds r={r:#x} s={s:#x} recid={recid}", int.from_bytes(rng.bytes(32), "little"), r, s, recid,
                    AGREE if 0 < r < N and 0 < s < N else None)
    d, z = rand(), int.from_bytes(rng.bytes(32), "little")
    r, s, recid = ref.sign(d, z, rand())
    for bad in list(range(4, 16)) + [127, 128, 254, 255]:
        add(f"recid {bad}", z, r, s, bad, None)
    return out
