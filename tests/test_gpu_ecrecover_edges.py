"""R on the GPU at its edges: phant_gpu_ecrecover_batch through the C ABI on signatures whose answer is known -- keys d G
from known d, the double multiplication's corners driven through (u1, u2), the x = r + n lift at its limits, every r / s /
recid boundary (tests/secp_corpus.py::crafted_signatures) -- each compared with tests/secp_ref.py and the oracle, every
address with keccak256(pub[1:])[12:]; batch sizes around the block size and past one pass of the grid-stride loop; device
pointers; NULL outputs; the argument checks and the counters; and a block of signed transactions through host.get_senders.
Outputs are filled with a poison byte before every call, so a byte the kernel fails to write is caught."""
import os

import numpy as np
import pytest

import secp_corpus as corpus
import secp_ref as ref
from secp_ref import N

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(os.environ.get("PHANT_GPU_ECRECOVER", "1") != "1", reason="PHANT_GPU_ECRECOVER=0")]

POISON = 0x5A


@pytest.fixture(scope="module")
def ctx():
    from phant_b200 import gpu
    c = gpu.Context(0)
    yield c
    c.close()


def run(ctx, hashes, sigs, pub=True, addr=True):
    n = len(hashes)
    h = np.frombuffer(b"".join(hashes), np.uint8)
    s = np.frombuffer(b"".join(sigs), np.uint8)
    p = np.full((n, 65), POISON, np.uint8) if pub else None
    a = np.full((n, 20), POISON, np.uint8) if addr else None
    ok = np.full(n, POISON, np.uint8)
    ctx.ecrecover_batch(h, s, n, p, a, ok)
    return p, a, ok


def assert_outputs(oracle, want, pub, addr, ok, label=lambda i: i):
    """want[i]: the 65-byte key or None.  Rejected: ok 0 and every output byte 0."""
    assert set(np.unique(ok).tolist()) <= {0, 1}
    for i, w in enumerate(want):
        assert ok[i] == (w is not None), label(i)
        if pub is not None:
            assert pub[i].tobytes() == (w if w is not None else bytes(65)), label(i)
        if addr is not None:
            assert addr[i].tobytes() == (oracle.keccak256(w[1:])[12:] if w is not None else bytes(20)), label(i)


@pytest.fixture(scope="module")
def crafted(oracle):
    """(labels, hashes, sigs, want): want checked against secp_ref and the oracle before any GPU call"""
    labels, hashes, sigs, want = [], [], [], []
    for label, h, sig, w in corpus.crafted_signatures():
        got = ref.recover(h, sig)
        assert got == oracle.ecrecover(h, sig), label
        assert w == corpus.AGREE or got == w, label
        labels.append(label), hashes.append(h), sigs.append(sig), want.append(got)
    return labels, hashes, sigs, want


def test_crafted_signatures(ctx, oracle, crafted):
    labels, hashes, sigs, want = crafted
    pub, addr, ok = run(ctx, hashes, sigs)
    assert_outputs(oracle, want, pub, addr, ok, lambda i: labels[i])
    assert sum(w is not None for w in want) > 400 and sum(w is None for w in want) > 100


@pytest.fixture(scope="module")
def mixed(oracle, crafted):
    """the crafted cases and 3,000 random tuples (small r, boundary s, recid > 3 mixed in), with the oracle's answers"""
    _, hashes, sigs, want = crafted
    hashes, sigs, want = list(hashes), list(sigs), list(want)
    rng = np.random.default_rng(31)
    for i in range(3000):
        r, s = int.from_bytes(rng.bytes(32), "big"), int.from_bytes(rng.bytes(32), "big")
        if i % 5 == 0:
            r %= 2 ** 128
        if i % 3 == 0:
            s %= N
        h, sig = rng.bytes(32), ref.sig65(r, s, int(rng.integers(0, 4)) if i % 23 else int(rng.integers(4, 256)))
        hashes.append(h), sigs.append(sig), want.append(oracle.ecrecover(h, sig))
    return hashes, sigs, want


def test_batch_sizes(ctx, oracle, mixed):
    """n = 1, 127, 129 around one block of 128 threads, and a batch past one pass of the grid-stride loop (the grid is
    capped at SMs x 8 blocks of 128 threads), tiled from the mixed cases"""
    import torch
    hashes, sigs, want = mixed
    cap = torch.cuda.get_device_properties(0).multi_processor_count * 8 * 128
    for n in (1, 127, 129):
        pub, addr, ok = run(ctx, hashes[7:7 + n], sigs[7:7 + n])
        assert_outputs(oracle, want[7:7 + n], pub, addr, ok)
    n = cap + 1000
    reps = -(-n // len(hashes))
    idx = np.arange(n) % len(hashes)
    pub, addr, ok = run(ctx, (hashes * reps)[:n], (sigs * reps)[:n])
    want_ok = np.array([w is not None for w in want], np.uint8)
    want_pub = np.stack([np.frombuffer(w if w is not None else bytes(65), np.uint8) for w in want])
    want_addr = np.stack([np.frombuffer(oracle.keccak256(w[1:])[12:] if w is not None else bytes(20), np.uint8) for w in want])
    assert (ok == want_ok[idx]).all() and (pub == want_pub[idx]).all() and (addr == want_addr[idx]).all()


def test_device_pointers(oracle, mixed):
    """PHANT_GPU_FLAG_DEVICE_PTRS: torch tensors in and out, nothing copied by the library"""
    import torch
    from phant_b200 import gpu
    hashes, sigs, want = mixed
    n = len(hashes)
    c = gpu.Context(0, gpu.FLAG_DEVICE_PTRS)
    try:
        d_h = torch.from_numpy(np.frombuffer(b"".join(hashes), np.uint8).copy()).cuda()
        d_s = torch.from_numpy(np.frombuffer(b"".join(sigs), np.uint8).copy()).cuda()
        d_pub = torch.full((n, 65), POISON, dtype=torch.uint8, device="cuda")
        d_addr = torch.full((n, 20), POISON, dtype=torch.uint8, device="cuda")
        d_ok = torch.full((n,), POISON, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()   # torch's copies and fills run on torch's stream, the library on its own
        c.reset_stats()
        c.ecrecover_batch(d_h, d_s, n, d_pub, d_addr, d_ok)
        c.synchronize()
        st = c.stats()
        assert st["launches"] == 1 and st["h2d_bytes"] == 0 and st["d2h_bytes"] == 0
        assert_outputs(oracle, want, d_pub.cpu().numpy(), d_addr.cpu().numpy(), d_ok.cpu().numpy())
    finally:
        c.close()


def test_null_outputs(ctx, oracle, mixed):
    """pubkeys65 = NULL or addresses20 = NULL: the other outputs are still right"""
    hashes, sigs, want = mixed
    pub, addr, ok = run(ctx, hashes, sigs, pub=False)
    assert pub is None
    assert_outputs(oracle, want, None, addr, ok)
    pub, addr, ok = run(ctx, hashes, sigs, addr=False)
    assert addr is None
    assert_outputs(oracle, want, pub, None, ok)


def test_arguments_and_counters(ctx, mixed):
    """n = 0 is a successful no-op; NULL ok (or inputs) with n > 0 is PHANT_GPU_E_INVALID with nothing launched or written;
    one call is one launch, 97 bytes per signature in and 65 + 20 + 1 out (less the outputs left NULL)"""
    from phant_b200 import gpu
    hashes, sigs, _ = mixed
    n = 300
    h = np.frombuffer(b"".join(hashes[:n]), np.uint8)
    s = np.frombuffer(b"".join(sigs[:n]), np.uint8)
    ctx.reset_stats()
    ctx.ecrecover_batch(None, None, 0, None, None, None)
    ctx.ecrecover_batch(h, s, 0, None, None, np.full(1, POISON, np.uint8))
    pub = np.full((n, 65), POISON, np.uint8)
    ok = np.full(n, POISON, np.uint8)
    for args in [(h, s, n, pub, None, None), (None, s, n, pub, None, ok), (h, None, n, pub, None, ok)]:
        with pytest.raises(gpu.PhantGpuError) as e:
            ctx.ecrecover_batch(*args)
        assert e.value.code == -1   # PHANT_GPU_E_INVALID
    assert (pub == POISON).all() and (ok == POISON).all()
    assert ctx.stats()["launches"] == 0
    for with_pub, with_addr in [(True, True), (False, True), (True, False)]:
        ctx.reset_stats()
        run(ctx, hashes[:n], sigs[:n], pub=with_pub, addr=with_addr)
        st = ctx.stats()
        assert st["launches"] == 1, st
        assert st["h2d_bytes"] == 97 * n, st
        assert st["d2h_bytes"] == (65 * with_pub + 20 * with_addr + 1) * n, st


# ---- a block of signed transactions through host.get_senders ----
def _rlp_bytes(b):
    return b if len(b) == 1 and b[0] < 0x80 else _rlp_header(0x80, len(b)) + b


def _rlp_int(i):
    return _rlp_bytes(i.to_bytes((i.bit_length() + 7) // 8, "big"))


def _rlp_header(base, n):
    if n < 56:
        return bytes([base + n])
    ln = n.to_bytes((n.bit_length() + 7) // 8, "big")
    return bytes([base + 55 + len(ln)]) + ln


def _rlp_list(items):
    payload = b"".join(items)
    return _rlp_header(0xC0, len(payload)) + payload


def _signed_transactions(oracle, chain_id, count, seed):
    """count transactions signed with secp_ref.sign by known keys -> (encoded, sender address).  Legacy with v = 27 / 28,
    EIP-155 legacy (v = 35 + 2 chain_id + parity), type 1 and type 2 (y parity in the body); always the low-s form.  Legacy
    transactions are signed in the EIP-155 form whenever the chain id is not 0, v = 27 / 28 included (the reference's
    TxSigner hashes them so)."""
    rng = np.random.default_rng(seed)
    keys = [int.from_bytes(rng.bytes(32), "big") % (N - 1) + 1 for _ in range(12)] + [1, N - 1]
    senders = [oracle.keccak256(ref.pubkey(d)[1:])[12:] for d in keys]
    out = []
    for i in range(count):
        j = int(rng.integers(0, len(keys)))
        to = rng.bytes(20)
        data = rng.bytes(int(rng.integers(0, 300)))
        nonce, gas, value = int(rng.integers(0, 2 ** 40)), int(rng.integers(21000, 2 ** 24)), int.from_bytes(rng.bytes(12), "big")
        fee = int(rng.integers(1, 2 ** 45))
        kind = i % 4
        if kind < 2:
            body = [_rlp_int(nonce), _rlp_int(fee), _rlp_int(gas), _rlp_bytes(to), _rlp_int(value), _rlp_bytes(data)]
            payload = _rlp_list(body + [_rlp_int(chain_id), _rlp_int(0), _rlp_int(0)])
        else:
            access = _rlp_list([_rlp_list([_rlp_bytes(rng.bytes(20)), _rlp_list([_rlp_bytes(rng.bytes(32))])])] if i % 8 == 3 else [])
            fees = [_rlp_int(fee)] if kind == 2 else [_rlp_int(fee // 3), _rlp_int(fee)]
            body = [_rlp_int(chain_id), _rlp_int(nonce)] + fees + [_rlp_int(gas), _rlp_bytes(to), _rlp_int(value), _rlp_bytes(data), access]
            payload = bytes([kind - 1]) + _rlp_list(body)
        z = int.from_bytes(oracle.keccak256(payload), "big")
        r, s, recid = ref.sign(keys[j], z, int.from_bytes(rng.bytes(32), "big") % (N - 1) + 1)
        if s > N // 2:
            s, recid = N - s, recid ^ 1
        assert recid < 2
        v = [27 + recid, 35 + 2 * chain_id + recid, recid, recid][kind]
        enc = _rlp_list(body + [_rlp_int(v), _rlp_int(r), _rlp_int(s)])
        out.append((enc if kind < 2 else bytes([kind - 1]) + enc, senders[j]))
    return out


@pytest.mark.parametrize("chain_id", [1, 2 ** 40 + 7])
def test_block_of_transactions(ctx, oracle, chain_id):
    from phant_b200 import host
    txs = _signed_transactions(oracle, chain_id, 500, seed=chain_id % 1000)
    got = host.get_senders(ctx, [t for t, _ in txs], chain_id=chain_id)
    assert [g if isinstance(g, bytes) else repr(g) for g in got] == [a for _, a in txs]
