"""The plain Python-integer model of secp256k1 (tests/secp_ref.py) pinned down: the reference's vectors and mainnet senders,
the oracle (oracle/secp256k1.c) on crafted and random signatures, and OpenSSL on signatures from random keys.  Also the
path coverage of the adversarial operand corpus (tests/secp_corpus.py) that the device and host checks of secp256k1.cuh
share.  CPU only."""
import numpy as np
import pytest

import secp_corpus as corpus
import secp_ref as ref
from secp_ref import N, P


def test_reference_vector_and_mainnet_senders(golden, oracle):
    from phant_b200 import host
    g = golden("ecrecover_kat.json")
    k = g["erecover"]
    assert ref.recover(bytes.fromhex(k["hash"]), bytes.fromhex(k["sig65"])).hex() == k["pubkey65"]
    for t in g["txs"]:
        payload, r, s, recid = host._tx_signing_parts(bytes.fromhex(t["encoded"]), t["chain_id"])
        pub = ref.recover(oracle.keccak256(payload), ref.sig65(r, s, recid))
        assert oracle.keccak256(pub[1:])[12:].hex() == t["sender"]


def test_group_law():
    """the generator is on the curve and has order n; the Jacobian ladder of mul() equals the affine definition"""
    assert ref.on_curve(ref.G) and ref.mul_affine(N, ref.G) is ref.INF and ref.mul_affine(N - 1, ref.G) == ref.neg(ref.G)
    rng = np.random.default_rng(5)
    for k in [0, 1, 2, 3, N - 2, N - 1, N, N + 1, 2 ** 255, 2 ** 256 - 1] + [int.from_bytes(rng.bytes(32), "big") for _ in range(12)]:
        want = ref.mul_affine(k, ref.G)
        assert ref.mul(k, ref.G) == want and ref.on_curve(want), k
    a, b = (int.from_bytes(rng.bytes(32), "big") % N for _ in range(2))
    A, B = ref.mul(a, ref.G), ref.mul(b, ref.G)
    assert ref.add(A, B) == ref.mul(a + b, ref.G) and ref.add(A, ref.neg(A)) is ref.INF and ref.double(A) == ref.add(A, A)
    for x in range(1, 40):
        y = ref.fp_sqrt((x ** 3 + 7) % P)
        assert y is None or ref.on_curve((x, y))


def test_sign_then_recover():
    rng = np.random.default_rng(6)
    for _ in range(40):
        d, k = (int.from_bytes(rng.bytes(32), "big") % (N - 1) + 1 for _ in range(2))
        z = int.from_bytes(rng.bytes(32), "big")
        r, s, recid = ref.sign(d, z, k)
        assert ref.recover(z.to_bytes(32, "big"), ref.sig65(r, s, recid)) == ref.pubkey(d)
        assert ref.recover(z.to_bytes(32, "big"), ref.sig65(r, N - s, recid ^ 1)) == ref.pubkey(d)
        assert ref.recover(z.to_bytes(32, "big"), ref.sig65(r, s, recid ^ 1)) not in (None, ref.pubkey(d))


def test_crafted_signatures_agree_with_the_oracle(oracle):
    n_key = 0
    for label, h, sig, want in corpus.crafted_signatures():
        got = ref.recover(h, sig)
        assert got == oracle.ecrecover(h, sig), label
        if want != corpus.AGREE:
            assert got == want, label
            n_key += want is not None
    assert n_key > 400


def test_random_tuples_agree_with_the_oracle(oracle):
    """recovery verifies nothing, so any (hash, r, s, recid) is a meaningful case"""
    rng = np.random.default_rng(9)
    outcomes = {True: 0, False: 0}
    for i in range(3000):
        r, s = int.from_bytes(rng.bytes(32), "big"), int.from_bytes(rng.bytes(32), "big")
        if i % 5 == 0:
            r %= 2 ** 128                # small r: recid 2 / 3 can lift
        if i % 7 == 0:
            s %= N
        recid = int(rng.integers(0, 4)) if i % 29 else int(rng.integers(4, 256))
        h, sig = rng.bytes(32), ref.sig65(r, s, recid)
        want = oracle.ecrecover(h, sig)
        assert ref.recover(h, sig) == want, (r, s, recid, h.hex())
        outcomes[want is not None] += 1
    assert outcomes[True] > 500 and outcomes[False] > 1000


def test_against_openssl():
    """OpenSSL's public keys and signatures: ref.pubkey equals OpenSSL's key, OpenSSL accepts ref.sign's signatures, and
    exactly one of recid 0 / 1 recovers the signer of an OpenSSL signature"""
    ec = pytest.importorskip("cryptography.hazmat.primitives.asymmetric.ec")
    from cryptography.hazmat.primitives import hashes, serialization
    from cryptography.hazmat.primitives.asymmetric.utils import Prehashed, decode_dss_signature, encode_dss_signature
    rng = np.random.default_rng(10)
    for _ in range(60):
        d = int.from_bytes(rng.bytes(32), "big") % (N - 1) + 1
        key = ec.derive_private_key(d, ec.SECP256K1())
        pub = key.public_key().public_bytes(serialization.Encoding.X962, serialization.PublicFormat.UncompressedPoint)
        assert ref.pubkey(d) == pub
        digest = rng.bytes(32)
        r, s = decode_dss_signature(key.sign(digest, ec.ECDSA(Prehashed(hashes.SHA256()))))
        got = [ref.recover(digest, ref.sig65(r, s, recid)) for recid in (0, 1)]
        assert got.count(pub) == 1, (r, s)
        r2, s2, _ = ref.sign(d, int.from_bytes(digest, "big"), int.from_bytes(rng.bytes(32), "big") % (N - 1) + 1)
        key.public_key().verify(encode_dss_signature(r2, s2), digest, ec.ECDSA(Prehashed(hashes.SHA256())))


@pytest.mark.parametrize("op", sorted(corpus.PATH_FLOORS))
def test_corpus_path_coverage(op):
    """every path of the fold and carry logic that uniform random operands almost never take is taken by at least the
    stated number of cases (fp_reduce k = 1, its folded value in [p, 2^256), sc_mul's third and fourth rounds, ...)"""
    counts = corpus.path_counts(op)
    for path, floor in corpus.PATH_FLOORS[op].items():
        assert counts[path] >= floor, (path, counts[path], floor)


def test_corpus_sizes():
    for op in corpus.OPS:
        assert len(corpus.cases(op)) >= corpus.SIZES[op]
