"""The trie builders at the encoders' size edges, on the GPU: every crafted case of tests/trie_edges.py (RLP header switches,
31 / 32 / 33-byte children, single-byte values, a root leaf under 32 bytes) through M alone, as one forest with awkward segment
shapes, and from device pointers; both sides of every layout switch of build_forest (slot vs general layout, single-CTA vs
per-level BFS); and accounts and slots of every width through S, the resident world state (root, reads, proofs) and T.  Every
root is compared with the C oracle and with helpers.py_mptize."""
import functools

import numpy as np
import pytest
import torch

import oracle_lib
import trie_edges
from helpers import py_mptize, secure_account_items
from phant_b200 import gpu, shard
from resident_state_model import ZERO32, Diff, StateModel, hashed_table, load_diff
from test_gpu_resident_state import apply_checked
from test_gpu_resident_state_proofs import proofs_checked
from test_gpu_resident_state_reads import read_checked
from test_gpu_resident_state_witness import witness_checked
from test_gpu_trie import gpu_state_root

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = gpu.Context(0)
    yield c
    c.close()


@functools.lru_cache(maxsize=None)
def corpus():
    return trie_edges.corpus()


def csr(kv):
    keys, koff = oracle_lib.csr([k for k, _ in kv], np.uint32)
    vals, voff = oracle_lib.csr([v for _, v in kv], np.uint64)
    return keys, koff, vals, voff


def gpu_root(ctx, kv):
    return ctx.mpt_root(*csr(kv)[:4], len(kv))


def gpu_forest(ctx, lists):
    flat = [x for l in lists for x in l]
    seg = np.zeros(len(lists) + 1, np.uint32)
    seg[1:] = np.cumsum([len(l) for l in lists])
    keys, koff, vals, voff = csr(flat)
    return ctx.mpt_roots(keys, koff, vals, voff, seg, len(lists))


def slot_layout_fits(kv):
    """build_forest's own test for the slot layout: no key a prefix of its successor, keys <= 64 bytes, values <= 3,072 bytes"""
    return (all(not kv[i + 1][0].startswith(kv[i][0]) for i in range(len(kv) - 1)) and max(len(k) for k, _ in kv) <= 64
            and max(len(v) for _, v in kv) <= 3072)


# ---------------------------------------------------------------- 1, 2: the corpus through M
def test_each_case_alone(ctx, oracle):
    for case in corpus():
        want = oracle.mptize(case.kv)
        assert want == py_mptize(oracle.keccak256, case.kv), case.name
        assert gpu_root(ctx, case.kv) == want, case.name


def boundary_segments():
    """adjacent segments whose keys are equal, or out of order, across the boundary (each segment is sorted on its own)"""
    return [[(b"\x10", b"a" * 40), (b"\x20", b"b")], [(b"\x20", b"c"), (b"\x30", b"d" * 33)],      # equal keys across
            [(b"\x90\x01", b"e" * 31), (b"\x90\x02", b"f")], [(b"\x10\x01", b"g"), (b"\x10\x02", b"h" * 32)],  # descending
            [(b"\x55", b"i")], [(b"\x55", b"i")]]                                                   # two equal one-key tries


def one_key_segments(rng, n):
    keys = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    lens = rng.choice([0, 1, 1, 2, 20, 26, 27, 28, 40], n)
    return [[(keys[i].tobytes(), rng.integers(0, 256, int(lens[i]), dtype=np.uint8).tobytes())] for i in range(n)]


def test_corpus_as_one_forest(ctx, oracle):
    """the whole corpus as one forest with empty segments between the cases (general layout: it holds prefix keys), then the
    cases the slot layout takes plus 100,000 one-key segments (slot layout), then that again with one prefix-key segment added
    (the whole forest falls back to the general layout)"""
    cases = [c.kv for c in corpus()]
    lists = [[]]
    for kv in cases:
        lists += [kv, []]
    lists += boundary_segments() + [[]]
    got = gpu_forest(ctx, lists)
    for i, kv in enumerate(lists):
        assert got[i] == oracle.mptize(kv), (i, len(kv))

    rng = np.random.default_rng(11)
    fits = [kv for kv in cases if slot_layout_fits(kv)]
    assert len(fits) >= 20
    lists = [[]] + fits[: len(fits) // 2] + [[]] + one_key_segments(rng, 100_000) + boundary_segments() + fits[len(fits) // 2:] + [[]]
    want = [oracle.mptize(kv) for kv in lists]
    prefix_seg = [(b"\x01", b"v" * 40), (b"\x01\x20", b"w"), (b"\x01\x30", b"x" * 50)]
    for extra in ([], [prefix_seg]):
        got = gpu_forest(ctx, lists + extra)
        assert got[len(lists):] == [oracle.mptize(kv) for kv in extra]
        bad = [i for i in range(len(lists)) if got[i] != want[i]]
        assert not bad, (len(extra), bad[:10], len(bad))


# ---------------------------------------------------------------- 3: both sides of build_forest's layout switches
def random_trie(rng, n, key_len, val_lens):
    """n distinct keys of key_len bytes (none a prefix of another), sorted, with values of the given lengths (cycled)"""
    keys = sorted({rng.integers(0, 256, key_len, dtype=np.uint8).tobytes() for _ in range(n)})
    return [(k, rng.integers(0, 256, int(val_lens[i % len(val_lens)]), dtype=np.uint8).tobytes()) for i, k in enumerate(keys)]


def comb(n_total, rng):
    """64-byte keys, the longest the slot layout takes: the all-zero key and one key per nibble position d whose nibble d is 1
    (a branch at every one of the 128 nibble depths under nibble 0, the deepest trie the slot layout builds), filled up to
    n_total keys with random 64-byte keys under nibbles 2..15"""
    keys = [bytes(64)]
    for d in range(128):
        k = bytearray(64)
        k[d // 2] = 0x10 if d % 2 == 0 else 0x01
        keys.append(bytes(k))
    fill = set()
    while len(fill) < n_total - len(keys):
        k = rng.integers(0, 256, 64, dtype=np.uint8)
        k[0] = int(rng.integers(0x20, 0x100))
        fill.add(k.tobytes())
    lens = [1, 5, 20, 31, 32, 40, 90]
    return [(k, rng.integers(0, 256, lens[i % len(lens)], dtype=np.uint8).tobytes()) for i, k in enumerate(sorted(keys + list(fill)))]


def test_layout_switches(ctx, oracle):
    """slot layout on one side, general on the other: 64 / 65-byte keys, 3,072 / 3,073-byte values, no prefix key / one; and
    the single-CTA BFS (slot layout, n <= 8,192) against the per-level BFS: 8,192 / 8,193 keys, and the 128-level comb at
    129, 8,192 and 8,193 keys"""
    rng = np.random.default_rng(5)
    base = random_trie(rng, 200, 20, [3, 40])
    switches = [  # (what, the tries, whether each fits the slot layout)
        ("key bytes 64 / 65", [random_trie(rng, 300, kl, [1, 31, 40, 3000]) for kl in (64, 65)], [True, False]),
        ("value bytes 3072 / 3073", [random_trie(rng, 300, 32, [vl, 1, 2, 30, 31, 100]) for vl in (3072, 3073)], [True, False]),
        ("no prefix key / one", [base, sorted(base + [(base[7][0][:9], b"p" * 33)])], [True, False]),
        ("keys 8192 / 8193", [random_trie(np.random.default_rng(6), n, 32, [1, 20, 33, 80]) for n in (8192, 8193)], [True, True]),
        ("comb 129 / 8192 / 8193", [comb(n, np.random.default_rng(7)) for n in (129, 8192, 8193)], [True, True, True]),
    ]
    assert [len(kv) for kv in switches[3][1] + switches[4][1]] == [8192, 8193, 129, 8192, 8193]
    for name, tries, fits in switches:
        assert [slot_layout_fits(kv) for kv in tries] == fits, name
        for kv in tries:
            assert gpu_root(ctx, kv) == oracle.mptize(kv), (name, len(kv))


def test_slot_layout_at_its_arena_bound_slow(ctx, oracle):
    """slow (about 2 GiB of values): 688,296 32-byte keys with 3,072-byte values, the most for which the slot layout's leaf
    arena (a stride of 3,120 bytes per leaf) stays within 2^31 bytes"""
    stride = (3072 + 32 + 16 + 15) & ~15
    n = (1 << 31) // stride
    assert stride * n <= 1 << 31 < stride * (n + 1)
    rng = np.random.default_rng(13)
    lead = np.unique(rng.integers(0, 2 ** 63, int(n * 1.01), dtype=np.uint64))
    lead = rng.permutation(lead)[:n]
    lead.sort()
    assert len(lead) == n
    keys = rng.integers(0, 256, (n, 32), dtype=np.uint8)
    keys[:, :8] = lead.astype(">u8").view(np.uint8).reshape(n, 8)
    vals = np.tile(rng.integers(0, 256, 3072, dtype=np.uint8), (n, 1))
    vals[:, :8] = np.arange(n, dtype=">u8").view(np.uint8).reshape(n, 8)
    koff = (np.arange(n + 1, dtype=np.uint64) * 32).astype(np.uint32)
    voff = np.arange(n + 1, dtype=np.uint64) * 3072
    keys, vals = keys.reshape(-1), vals.reshape(-1)
    assert ctx.mpt_root(keys, koff, vals, voff, n) == oracle.mptize_csr(keys, koff, vals, voff)


# ---------------------------------------------------------------- 4: device pointers
def test_device_pointers(ctx, oracle):
    """the corpus through phant_gpu_mpt_root with FLAG_DEVICE_PTRS, from torch tensors: key and value bytes 16-byte aligned and
    at odd offsets; equal to the host-pointer call and to the oracle"""
    dev = torch.device("cuda", 0)

    def at(a, shift):
        buf = torch.zeros(a.size + shift + 16, dtype=torch.uint8, device=dev)
        buf[shift:shift + a.size] = torch.from_numpy(a.copy()).to(dev)
        return buf[shift:]

    done = 0
    for case in corpus():
        keys, koff, vals, voff = csr(case.kv)
        host_root = ctx.mpt_root(keys, koff, vals, voff, len(case.kv))
        assert host_root == oracle.mptize(case.kv), case.name
        dko, dvo = torch.from_numpy(koff.copy()).to(dev), torch.from_numpy(voff.copy()).to(dev)
        for ks, vs in ((0, 0), (1, 3), (7, 1), (0, 5), (3, 0)):
            dk, dv = at(keys, ks), at(vals, vs)
            torch.cuda.synchronize()  # torch's copies run on torch's stream, the library on its own
            ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
            try:
                got = ctx.mpt_root(dk, dko, dv, dvo, len(case.kv))
            finally:
                ctx.set_flags(0)
            assert got == host_root, (case.name, ks, vs)
            done += 1
    assert done == 5 * len(corpus())


# ---------------------------------------------------------------- 5: accounts and slots of every width
NONCES = [0, 1, 0x7f, 0x80, 0xff, 0x100, 2 ** 56 - 1, 2 ** 56, 2 ** 63, 2 ** 64 - 1]
BALANCES = [0, 1, 0x7f, 0x80, 2 ** 248 - 1, 2 ** 248, 2 ** 255, 2 ** 256 - 1]


def slot_values(rng):
    """every value length from 1 to 32 bytes, each with a first byte below 0x80 and one at or above it (32-byte words)"""
    out = []
    for n in range(1, 33):
        for first in (int(rng.integers(1, 0x80)), int(rng.integers(0x80, 0x100))):
            out.append(bytes(32 - n) + bytes([first]) + rng.integers(0, 256, n - 1, dtype=np.uint8).tobytes())
    return out


def width_accounts(rng):
    """one account per (nonce, balance) pair; empty and non-empty code; slots cycling through every value width, plus one
    account holding all of them and a zero slot (no slot)"""
    vals = slot_values(rng)
    accounts, j = [], 0
    for i, (nonce, bal) in enumerate((x, y) for x in NONCES for y in BALANCES):
        storage = {}
        for _ in range(i % 4):
            storage[rng.integers(0, 256, 32, dtype=np.uint8).tobytes().hex()] = vals[j % len(vals)].hex()
            j += 1
        if i == 17:
            storage.update({rng.integers(0, 256, 32, dtype=np.uint8).tobytes().hex(): v.hex() for v in vals})
            storage[rng.integers(0, 256, 32, dtype=np.uint8).tobytes().hex()] = ZERO32.hex()
        code = rng.integers(0, 256, int(rng.choice([1, 33, 600])), dtype=np.uint8).tobytes() if i % 3 else b""
        accounts.append({"address": rng.integers(0, 256, 20, dtype=np.uint8).tobytes().hex(), "nonce": nonce, "balance": "%064x" % bal,
                         "code": code.hex(), "storage": storage})
    return accounts


def flat_accounts(accounts):
    n = len(accounts)
    addr = np.frombuffer(b"".join(bytes.fromhex(a["address"]) for a in accounts), np.uint8)
    nonce = np.array([a["nonce"] for a in accounts], np.uint64)
    bal = np.frombuffer(b"".join(bytes.fromhex(a["balance"]) for a in accounts), np.uint8)
    code, coff = oracle_lib.csr([bytes.fromhex(a["code"]) for a in accounts])
    sk = [bytes.fromhex(k) for a in accounts for k in a["storage"]]
    sv = [bytes.fromhex(v) for a in accounts for v in a["storage"].values()]
    soff = np.zeros(n + 1, np.uint64)
    soff[1:] = np.cumsum([len(a["storage"]) for a in accounts])
    return addr, nonce, bal, code, coff, np.frombuffer(b"".join(sk), np.uint8), np.frombuffer(b"".join(sv), np.uint8), soff


def test_account_widths_through_s(ctx, oracle):
    """state_root, and state_subtree_roots combined over 1, 4 and 16 simulated ranks, equal oracle.state_root and the
    secure_account_items + py_mptize root"""
    accounts = width_accounts(np.random.default_rng(31))
    want = oracle.state_root(accounts)
    assert want == py_mptize(oracle.keccak256, secure_account_items(oracle.keccak256, oracle.mptize, accounts))
    assert ctx.state_root(len(accounts), *flat_accounts(accounts)) == want
    assert gpu_state_root(ctx, accounts) == want
    top = [oracle.keccak256(bytes.fromhex(a["address"]))[0] >> 4 for a in accounts]
    for world in (1, 4, 16):
        refs, mask = np.zeros((16, 32), np.uint8), 0
        for rank in range(world):
            mine = [a for a, t in zip(accounts, top) if shard.nibble_owner(t, world) == rank]
            if not mine:
                continue
            r, m = ctx.state_subtree_roots(len(mine), *flat_accounts(mine))
            assert mask & m == 0
            refs, mask = refs + r, mask | m
        assert bin(mask).count("1") >= 2
        assert oracle.keccak256(shard.root_branch_rlp(refs, mask)) == want, world


def test_account_widths_through_the_resident_state(ctx, oracle):
    """the same state loaded into the resident world state: the root, every nonce, balance and slot value read back, proofs
    that V accepts with the model's values; then a block that moves every account to other widths, whose witness gives T the
    root apply gives"""
    rng = np.random.default_rng(32)
    accounts = width_accounts(rng)
    table = hashed_table(oracle.keccak256, accounts)
    st = ctx.resident_state()
    m = StateModel(oracle)
    assert apply_checked(st, m, load_diff(table)) == oracle.state_root(accounts)
    akeys = sorted(m.acc) + [rng.integers(0, 256, 32, dtype=np.uint8).tobytes()]
    slots = [(i, sk) for i, k in enumerate(akeys) if k in m.acc for sk in m.acc[k].storage]
    slots.append((0, rng.integers(0, 256, 32, dtype=np.uint8).tobytes()))
    read_checked(st, m, akeys, slots)
    proofs_checked(ctx, oracle, st, m, akeys, slots)

    vals = slot_values(rng)
    d = Diff()
    for i, k in enumerate(sorted(m.acc)):
        a = m.acc[k]
        d.accounts.append((k, 0, NONCES[(NONCES.index(a.nonce) + 3) % len(NONCES)],
                           int.to_bytes(BALANCES[(BALANCES.index(int.from_bytes(a.balance, "big")) + 5) % len(BALANCES)], 32, "big"),
                           a.code_hash))
        for j, sk in enumerate(sorted(a.storage)):
            d.slots.append((i, sk, ZERO32 if j % 3 == 2 else vals[(i + j) % len(vals)]))
        d.slots.append((i, rng.integers(0, 256, 32, dtype=np.uint8).tobytes(), vals[(7 * i) % len(vals)]))
    witness_checked(ctx, oracle, st, m, d)
    akeys = sorted(m.acc)
    slots = [(i, sk) for i, k in enumerate(akeys) for sk in m.acc[k].storage]
    read_checked(st, m, akeys, slots)
    proofs_checked(ctx, oracle, st, m, akeys, slots)
    st.close()
