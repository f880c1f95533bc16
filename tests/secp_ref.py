"""secp256k1 in plain Python integers: the reference the sender-recovery tests hold the CUDA code and the oracle to.

No limbs, no tricks: field and scalar arithmetic are Python's `%` and `pow`, points are affine pairs (None is the point at
infinity), scalar multiplication is double-and-add.  recover() applies the SEC 1 v2 section 4.1.6 rules stated in the
header of phant_b200/csrc/secp256k1.cuh:
  0 < r < n, 0 < s < n, recid <= 3;  x = r (+ n if recid & 2) must be < p and on the curve;  y parity = recid & 1;
  Q = u1 G + u2 R with u1 = -z / r, u2 = s / r (mod n);  Q at infinity fails."""

P = 2 ** 256 - 0x1000003D1
N = 0xFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFFEBAAEDCE6AF48A03BBFD25E8CD0364141
C = 0x1000003D1                      # 2^256 - p
K = 2 ** 256 - N                     # 2^256 - n
GX = 0x79BE667EF9DCBBAC55A06295CE870B07029BFCDB2DCE28D959F2815B16F81798
GY = 0x483ADA7726A3C4655DA4FBFC0E1108A8FD17B448A68554199C47D08FFB10D4B8
G = (GX, GY)
INF = None


# ---- field and scalars ----
def fp_inv(a):
    return pow(a, -1, P)


def fp_sqrt(a):
    """a square root of a mod p, or None when a is not a square (p = 3 mod 4: the root is a^((p+1)/4))"""
    y = pow(a, (P + 1) // 4, P)
    return y if y * y % P == a % P else None


def sc_inv(a):
    return pow(a, -1, N)


# ---- points ----
def on_curve(pt):
    return pt is INF or (pt[1] * pt[1] - pt[0] ** 3 - 7) % P == 0


def neg(pt):
    return INF if pt is INF else (pt[0], (-pt[1]) % P)


def double(pt):
    if pt is INF or pt[1] == 0:
        return INF
    x, y = pt
    lam = 3 * x * x * fp_inv(2 * y) % P
    x3 = (lam * lam - 2 * x) % P
    return (x3, (lam * (x - x3) - y) % P)


def add(p1, p2):
    if p1 is INF:
        return p2
    if p2 is INF:
        return p1
    if p1[0] == p2[0]:
        return double(p1) if p1[1] == p2[1] else INF
    lam = (p2[1] - p1[1]) * fp_inv(p2[0] - p1[0]) % P
    x3 = (lam * lam - p1[0] - p2[0]) % P
    return (x3, (lam * (p1[0] - x3) - p1[1]) % P)


def mul_affine(k, pt):
    """k * pt for any integer k >= 0: double-and-add from the top bit, the definition mul() is checked against"""
    acc = INF
    for bit in bin(k)[2:] if k else "":
        acc = double(acc)
        if bit == "1":
            acc = add(acc, pt)
    return acc


def mul(k, pt):
    """k * pt, the same ladder as mul_affine with the accumulator in Jacobian coordinates (x = X / Z^2, y = Y / Z^3) so that
    it takes one inversion instead of one per step; about ten times faster in Python"""
    if pt is INF:
        return INF
    X, Y, Z = 0, 1, 0
    for bit in bin(k)[2:] if k else "":
        if Z:                                     # doubling; y = 0 does not occur on this curve (its order is odd)
            S, M = 4 * X * Y * Y % P, 3 * X * X % P
            X2 = (M * M - 2 * S) % P
            X, Y, Z = X2, (M * (S - X2) - 8 * Y ** 4) % P, 2 * Y * Z % P
        if bit == "1":
            if not Z:
                X, Y, Z = pt[0], pt[1], 1
                continue
            Z2 = Z * Z % P
            H, R = (pt[0] * Z2 - X) % P, (pt[1] * Z2 * Z - Y) % P
            if H == 0:                             # the accumulator is pt or -pt
                if R:
                    X, Y, Z = 0, 1, 0
                else:
                    X, Y = double(pt)
                    Z = 1
                continue
            H2 = H * H % P
            H3, V = H2 * H % P, X * H2 % P
            X3 = (R * R - H3 - 2 * V) % P
            X, Y, Z = X3, (R * (V - X3) - Y * H3) % P, Z * H % P
    if not Z:
        return INF
    zi = fp_inv(Z)
    return (X * zi * zi % P, Y * zi ** 3 % P)


def lift_x(x, parity):
    """the curve point with abscissa x and y = parity (mod 2), or None when x is not the abscissa of a point"""
    if not 0 <= x < P:
        return None
    y = fp_sqrt((x ** 3 + 7) % P)
    if y is None:
        return None
    return (x, y if y & 1 == parity else P - y)


def encode(pt):
    """65-byte uncompressed public key 0x04 || X || Y"""
    return b"\x04" + pt[0].to_bytes(32, "big") + pt[1].to_bytes(32, "big")


def pubkey(d):
    return encode(mul(d % N, G))


# ---- ECDSA ----
def recover(hash32, sig65):
    """hash32 = message hash, sig65 = r || s || recid -> the 65-byte public key, or None when no key is recovered"""
    r = int.from_bytes(sig65[:32], "big")
    s = int.from_bytes(sig65[32:64], "big")
    recid = sig65[64]
    if recid > 3 or not 0 < r < N or not 0 < s < N:
        return None
    R = lift_x(r + N if recid & 2 else r, recid & 1)
    if R is None:
        return None
    z = int.from_bytes(hash32, "big") % N
    rinv = sc_inv(r)
    u1, u2 = -z * rinv % N, s * rinv % N
    Q = add(mul(u1, G), mul(u2, R))
    return None if Q is INF else encode(Q)


def sign(d, z, k):
    """ECDSA signature of the hash z (an integer < 2^256) with key d and nonce k -> (r, s, recid); recid tells recover()
    which of the up to four candidate points R was.  s is returned as computed (either half): callers pick the form."""
    R = mul(k % N, G)
    if R is INF:
        raise ValueError("k = 0 mod n")
    r = R[0] % N
    s = sc_inv(k) * (z + r * d) % N
    if r == 0 or s == 0:
        raise ValueError("degenerate nonce")
    return r, s, (R[1] & 1) | (2 if R[0] >= N else 0)


def sig65(r, s, recid):
    return r.to_bytes(32, "big") + s.to_bytes(32, "big") + bytes([recid])
