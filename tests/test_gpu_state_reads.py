"""P: pre-state reads on the GPU (phant_gpu_read_state) -- against the fixture tables themselves, against the existing
two-step procedure (W over accounts, storage roots decoded on the host, W over slots), against the CPU statement
(tests/state_read_oracle.py) on crafted values, in both pointer modes, and on the C5 block witnesses."""
import numpy as np
import pytest

import oracle_lib
from helpers import rlp_list, rlp_str
from state_read_oracle import (CODE_EMPTY, CODE_MISSING, EMPTY_CODE_HASH, check_against_fixture, decode_account, fixture_reads,
                               fixture_roots, read_state)

pytestmark = pytest.mark.gpu

EMPTY_ROOT = bytes.fromhex("56e81f171bcc55a6ff8345e692c0f86e5b48e01b996cadc001622fb5e363b421")
FIELDS = ("account_status", "nonce", "balance32", "storage_root32", "code_hash32", "code_index", "slot_status", "slot_vals32")


@pytest.fixture(scope="module")
def ctx():
    from phant_b200 import gpu
    c = gpu.Context(0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def fixture(oracle, golden):
    return fixture_reads(oracle, golden("fixture_states.json.gz"))


def _u8(b):
    return np.frombuffer(bytes(b), np.uint8).copy()


def empty_outputs(na, ns, fill=0x77):
    return dict(account_status=np.full(na, fill, np.uint8), nonce=np.full(na, fill, np.uint64), balance32=np.full((na, 32), fill, np.uint8),
                storage_root32=np.full((na, 32), fill, np.uint8), code_hash32=np.full((na, 32), fill, np.uint8),
                code_index=np.full(na, fill, np.uint32), slot_status=np.full(ns, fill, np.uint8), slot_vals32=np.full((ns, 32), fill, np.uint8))


def gpu_read(ctx, nodes, node_off, roots32, akeys, skeys=None, sacc=None, codes=(), want=FIELDS):
    """host-pointer P call; the requested outputs come back pre-filled with 0x77, so anything left unwritten shows"""
    na, ns = akeys.size // 32, 0 if skeys is None else skeys.size // 32
    cdata, coff = oracle_lib.csr(list(codes), np.uint64) if len(codes) else (None, None)
    out = {k: v for k, v in empty_outputs(na, ns).items() if k in want}
    ctx.read_state(len(node_off) - 1, nodes, node_off, na, akeys, roots32, roots32.size // 32, ns, skeys, sacc, len(codes), cdata, coff, **out)
    return out


def assert_same(got, want, fields=FIELDS):
    for k in fields:
        assert (np.asarray(got[k]) == np.asarray(want[k])).all(), (k, np.nonzero(np.asarray(got[k]) != np.asarray(want[k]))[0][:10])


# ---- 1. the fixture tables ------------------------------------------------------------------------------------------------
def test_fixture_tables_and_state_root_round_trip(ctx, oracle, golden, fixture):
    """all 91 fixture tables in ONE call: the expectations come from the tables, not from the oracle; the values read rebuild
    every table's root through phant_gpu_state_root"""
    r = fixture
    got = gpu_read(ctx, r["nodes"], r["node_off"], r["roots32"], r["account_keys32"], r["slot_keys32"], r["slot_account"], r["codes"])
    check_against_fixture(r, got, r["codes"])
    assert (got["account_status"] == 1).sum() >= 1100 and (got["slot_status"] == 1).sum() >= 70
    # round trip: what was read, handed to S, gives the fixture root again
    g = golden("fixture_states.json.gz")
    root_of = fixture_roots(g)
    per_table = {}
    for i, w in enumerate(r["account_want"]):
        if w is not None:
            per_table.setdefault(w[0], []).append((i, w[1]))
    slots_of = {}
    for j, (st, _, pre) in enumerate(r["slot_want"]):
        if st == 1:
            slots_of.setdefault(int(r["slot_account"][j]), []).append((pre.rjust(32, b"\x00"), got["slot_vals32"][j].tobytes()))
    assert len(per_table) == sum(1 for a in g["tables"].values() if a)
    for tab, accts in per_table.items():
        n = len(accts)
        addr = _u8(b"".join(bytes.fromhex(a["address"]) for _, a in accts))
        nonce = np.array([got["nonce"][i] for i, _ in accts], np.uint64)
        bal = np.ascontiguousarray(np.stack([got["balance32"][i] for i, _ in accts]))
        code, coff = oracle_lib.csr([bytes(r["codes"][got["code_index"][i]]) if got["code_index"][i] != CODE_EMPTY else b"" for i, _ in accts], np.uint64)
        sk, sv, soff = [], [], [0]
        for i, _ in accts:
            for k, v in slots_of.get(i, []):
                sk.append(k); sv.append(v)
            soff.append(len(sk))
        skeys = _u8(b"".join(sk) or bytes(1))
        svals = _u8(b"".join(sv) or bytes(1))
        root = ctx.state_root(n, addr, nonce, bal, code, coff, skeys, svals, np.array(soff, np.uint64))
        assert root.hex() == root_of[tab], tab
    # and the CPU statement agrees on every output
    assert_same(got, read_state(oracle, r["nodes"], r["node_off"], r["roots32"], r["account_keys32"], r["slot_keys32"], r["slot_account"],
                                r["codes"]))


# ---- 2. the existing two-step procedure ------------------------------------------------------------------------------------
def test_agrees_with_witness_walk_and_host_decoded_roots(ctx, fixture):
    r = fixture
    nodes, off, nn = r["nodes"], r["node_off"], r["n_nodes"]
    na, ns = r["account_keys32"].size // 32, r["slot_keys32"].size // 32
    got = gpu_read(ctx, nodes, off, r["roots32"], r["account_keys32"], r["slot_keys32"], r["slot_account"], r["codes"])
    st, vo, vl = np.zeros(na, np.uint8), np.zeros(na, np.uint64), np.zeros(na, np.uint32)
    ctx.verify_witness(nn, nodes, off, na, r["account_keys32"], r["roots32"], na, None, st, vo, vl)
    assert (got["account_status"] == st).all()
    roots = np.zeros((na, 32), np.uint8)
    for i in np.nonzero(st == 1)[0]:
        roots[i] = _u8(decode_account(nodes[int(vo[i]):int(vo[i]) + int(vl[i])].tobytes())[2])
    assert (roots == got["storage_root32"]).all()
    acc = r["slot_account"].astype(np.int64)
    walk = np.nonzero(st[acc] == 1)[0]
    sst, svo, svl = np.zeros(len(walk), np.uint8), np.zeros(len(walk), np.uint64), np.zeros(len(walk), np.uint32)
    ctx.verify_witness(nn, nodes, off, len(walk), np.ascontiguousarray(r["slot_keys32"].reshape(-1, 32)[walk]),
                       np.ascontiguousarray(roots[acc[walk]]), len(walk), None, sst, svo, svl)
    assert (got["slot_status"][walk] == sst).all()
    for j, i in enumerate(walk):
        if sst[j] == 1:
            payload = nodes[int(svo[j]):int(svo[j]) + int(svl[j])].tobytes()
            assert got["slot_vals32"][i].tobytes() == rlp_payload(payload).rjust(32, b"\x00")
    assert ns > len(walk)  # some slots belong to absent accounts: status 2 without a walk
    assert (got["slot_status"][np.nonzero(st[acc] == 2)[0]] == 2).all()


def rlp_payload(b):
    if b[0] < 0x80:
        return b
    assert b[0] <= 0xB7
    return b[1:1 + b[0] - 0x80]


# ---- 3. crafted values and incomplete node sets against the CPU statement -------------------------------------------------
def crafted_witness(oracle):
    """accounts with every body mutation class, a storage trie holding every slot-value mutation class, embedded storage
    leaves, an empty storage root, codes missing and repeated.  -> the tries and their key/values.  (reads_of reads only an
    evenly spaced sample of about 40 of the storage trie's slots on the GPU; every slot-value class goes through the same
    decoder compiled as host code in tests/test_state_read_header_host.py.)"""
    from test_state_read_header_host import structural_account_mutations, valid_slots, slot_mutations, header_mutations
    rng = np.random.default_rng(5)
    # storage tries: every slot payload class under one root; 1-byte values in leaves short enough to be embedded
    payloads = list({p: 1 for p in valid_slots() + slot_mutations(rng) if len(p)})
    skv = sorted((oracle.keccak256(b"slot %d" % i), p) for i, p in enumerate(payloads))
    strie = oracle.trie(skv)
    ekv = [(bytes(31) + bytes([i]), bytes([1 + i])) for i in range(20)]  # keys share 62 nibbles: leaves of 3 bytes, embedded
    etrie = oracle.trie(ekv)
    codes = [b"\x60\x00", b"\x60\x01\x60\x02", b"\x60\x00", b"code never sent"]  # a repeated code, and one left out below
    good = lambda root, code: rlp_list([b"\x01", rlp_str(b"\x0a"), rlp_str(root), rlp_str(code)])
    bodies = [good(strie.root(), oracle.keccak256(codes[0])), good(etrie.root(), oracle.keccak256(codes[1])),
              good(EMPTY_ROOT, EMPTY_CODE_HASH), good(strie.root(), oracle.keccak256(codes[3]))]
    base = bodies[0]
    bodies += structural_account_mutations(rng) + [m for m in header_mutations(base)[::7] if m and m[0] >= 0xC0]
    akv = sorted({oracle.keccak256(b"acct %d" % i): b for i, b in enumerate(bodies)}.items())
    atrie = oracle.trie(akv)
    key_of = {b: k for k, b in akv}
    return dict(strie=strie, skv=skv, etrie=etrie, ekv=ekv, codes=codes[:3], atrie=atrie, akv=akv, bodies=bodies, key_of=key_of)


def reads_of(oracle, c):
    """every account; under EVERY account (so each account status reaches its slots) about 40 evenly spaced slots of the
    mutation storage trie, every slot of the embedded-leaf trie and an absent slot; an absent account"""
    akeys = [k for k, _ in c["akv"]] + [oracle.keccak256(b"no such account")]
    skeys, sacc = [], []
    for i in range(len(akeys)):
        for k, _ in c["skv"][:: max(1, len(c["skv"]) // 40)] + c["ekv"] + [(oracle.keccak256(b"absent slot"), None)]:
            skeys.append(k); sacc.append(i)
    return _u8(b"".join(akeys)), _u8(b"".join(skeys)), np.array(sacc, np.uint32)


def node_set(*tries_and_keys):
    nodes = {}
    for trie, keys in tries_and_keys:
        for k in keys:
            for nd in trie.prove(k):
                nodes[nd] = 1
    return list(nodes)


def run_both(ctx, oracle, node_list, root, akeys, skeys, sacc, codes):
    data, off = oracle_lib.csr(node_list, np.uint64)
    data = np.concatenate([data, np.zeros(64, np.uint8)])
    got = gpu_read(ctx, data, off, _u8(root), akeys, skeys, sacc, codes)
    want = read_state(oracle, data, off, _u8(root), akeys, skeys, sacc, codes)
    assert_same(got, want)
    return got


def test_crafted_values_and_incomplete_sets_vs_oracle(ctx, oracle):
    c = crafted_witness(oracle)
    akeys, skeys, sacc = reads_of(oracle, c)
    na = akeys.size // 32
    all_a = [k for k, _ in c["akv"]] + [oracle.keccak256(b"no such account")]
    all_s = [k for k, _ in c["skv"]] + [oracle.keccak256(b"absent slot")]
    all_e = [k for k, _ in c["ekv"]] + [oracle.keccak256(b"absent slot")]
    full = node_set((c["atrie"], all_a), (c["strie"], all_s), (c["etrie"], all_e))
    root = c["atrie"].root()
    got = run_both(ctx, oracle, full, root, akeys, skeys, sacc, c["codes"])
    st = got["account_status"]
    i_s, i_e, i_x, i_m = (all_a.index(c["key_of"][c["bodies"][j]]) for j in range(4))
    assert st[i_s] == st[i_e] == st[i_x] == st[i_m] == 1 and st[-1] == 2
    assert (st == 0).sum() >= 20  # the mutated bodies
    assert got["code_index"][i_s] in (0, 2) and got["code_index"][i_e] == 1 and got["code_index"][i_x] == CODE_EMPTY
    assert got["code_index"][i_m] == CODE_MISSING
    per = len(skeys) // 32 // na
    sst = got["slot_status"].reshape(na, per)
    assert {0, 1, 2} <= set(np.unique(sst[i_s]).tolist())               # the slot-value mutation classes
    assert (sst[i_x] == 2).all() and not got["slot_vals32"].reshape(na, per, 32)[i_x].any()  # empty storage root
    assert (sst[st == 0] == 0).all() and (sst[-1] == 2).all()
    emb = slice(per - len(c["ekv"]) - 1, per - 1)                       # the embedded leaves under the etrie account
    assert (sst[i_e, emb] == 1).all()
    assert got["slot_vals32"].reshape(na, per, 32)[i_e, emb, 31].tolist() == [1 + i for i in range(20)]
    # n_codes = 0: every non-empty code hash is missing
    got0 = run_both(ctx, oracle, full, root, akeys, skeys, sacc, ())
    assert got0["code_index"][i_s] == CODE_MISSING and got0["code_index"][i_x] == CODE_EMPTY
    # a storage node removed: the slots under it lack a node, the account is still present
    leaf = c["strie"].prove(c["skv"][0][0])[-1]
    got = run_both(ctx, oracle, [nd for nd in full if nd != leaf], root, akeys, skeys, sacc, c["codes"])
    assert got["account_status"][i_s] == 1 and got["slot_status"].reshape(na, per)[i_s, 0] == 3
    # an account leaf removed: that account and all its slots lack a node
    aleaf = c["atrie"].prove(all_a[i_s])[-1]
    got = run_both(ctx, oracle, [nd for nd in full if nd != aleaf], root, akeys, skeys, sacc, c["codes"])
    assert got["account_status"][i_s] == 3 and (got["slot_status"].reshape(na, per)[i_s] == 3).all()
    # an account leaf corrupted: it no longer hashes to its reference -> the same
    bad = bytearray(aleaf); bad[-1] ^= 1
    got = run_both(ctx, oracle, [bytes(bad) if nd == aleaf else nd for nd in full], root, akeys, skeys, sacc, c["codes"])
    assert got["account_status"][i_s] == 3 and (got["slot_status"].reshape(na, per)[i_s] == 3).all()
    assert got["account_status"][i_e] == 1


# ---- 4. pointer modes, NULL outputs, argument errors, launch counts ---------------------------------------------------------
def device_read(ctx, r, codes, want=FIELDS):
    import torch
    from phant_b200 import gpu
    na, ns = r["account_keys32"].size // 32, r["slot_keys32"].size // 32
    cdata, coff = oracle_lib.csr(list(codes), np.uint64)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8) if a.dtype != np.uint64 else a.view(np.int64)).cuda()
    d = dict(nodes=t(r["nodes"]), off=torch.from_numpy(r["node_off"].view(np.int64)).cuda(), akeys=t(r["account_keys32"]), roots=t(r["roots32"]),
             skeys=t(r["slot_keys32"]), sacc=torch.from_numpy(r["slot_account"].view(np.int32)).cuda(),
             codes=t(np.concatenate([cdata, np.zeros(64, np.uint8)])), coff=torch.from_numpy(coff.view(np.int64)).cuda())
    host = empty_outputs(na, ns)
    out = {k: torch.from_numpy(v.view(np.uint8).reshape(-1)).cuda() for k, v in host.items() if k in want}
    torch.cuda.synchronize()
    ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
    try:
        ctx.read_state(r["n_nodes"], d["nodes"], d["off"], na, d["akeys"], d["roots"], r["roots32"].size // 32, ns, d["skeys"], d["sacc"],
                       len(codes), d["codes"], d["coff"], nodes_bytes=int(r["node_off"][-1]), codes_bytes=int(coff[-1]), **out)
        ctx.synchronize()
    finally:
        ctx.set_flags(0)
    return {k: v.cpu().numpy().view(host[k].dtype).reshape(host[k].shape) for k, v in out.items()}


def test_host_and_device_pointers_and_null_outputs(ctx, fixture):
    r = fixture
    args = (r["nodes"], r["node_off"], r["roots32"], r["account_keys32"], r["slot_keys32"], r["slot_account"], r["codes"])
    full = gpu_read(ctx, *args)
    assert_same(device_read(ctx, r, r["codes"]), full)
    for want in (("slot_status",), ("slot_vals32", "nonce"), ("code_index", "balance32"), ()):
        part = gpu_read(ctx, *args, want=want)
        assert set(part) == set(want)
        assert_same(part, full, want)
    assert_same(device_read(ctx, r, r["codes"], want=("slot_vals32", "account_status")), full, ("slot_vals32", "account_status"))


def test_device_pointers_out_of_range_slot_account(ctx, fixture):
    """device pointers are not validated: a slot whose account index is out of range gets status 0 and value 0 (and no
    read past the account records); every other read is unchanged"""
    r = fixture
    na, ns = r["account_keys32"].size // 32, r["slot_keys32"].size // 32
    full = gpu_read(ctx, r["nodes"], r["node_off"], r["roots32"], r["account_keys32"], r["slot_keys32"], r["slot_account"], r["codes"])
    bad = dict(r)
    bad["slot_account"] = r["slot_account"].copy()
    hit = [0, ns // 2, ns - 1]
    bad["slot_account"][hit] = [na, na + 1000, 0xFFFFFFFF]
    assert (full["slot_status"][hit] != 0).any()
    got = device_read(ctx, bad, r["codes"])
    assert (got["slot_status"][hit] == 0).all() and not got["slot_vals32"][hit].any()
    keep = np.setdiff1d(np.arange(ns), hit)
    assert (got["slot_status"][keep] == full["slot_status"][keep]).all() and (got["slot_vals32"][keep] == full["slot_vals32"][keep]).all()
    assert_same(got, full, FIELDS[:6])


def test_invalid_arguments_launch_nothing(ctx, fixture):
    from phant_b200 import gpu
    r = fixture
    args = dict(nodes=r["nodes"], node_off=r["node_off"], roots32=r["roots32"], akeys=r["account_keys32"], skeys=r["slot_keys32"],
                sacc=r["slot_account"], codes=r["codes"])

    def call(**kw):
        a = {**args, **kw}
        return gpu_read(ctx, a["nodes"], a["node_off"], a["roots32"], a["akeys"], a["skeys"], a["sacc"], a["codes"])
    ctx.reset_stats()
    bad_off = r["node_off"].copy(); bad_off[5] = bad_off[6] + 1
    na = r["account_keys32"].size // 32
    bad_acc = r["slot_account"].copy(); bad_acc[-1] = na
    for kw in (dict(node_off=bad_off), dict(sacc=bad_acc), dict(roots32=np.ascontiguousarray(r["roots32"][:64]))):
        with pytest.raises(gpu.PhantGpuError) as e:
            call(**kw)
        assert e.value.code == -1
    # a bad code CSR
    cdata, coff = oracle_lib.csr(list(r["codes"]), np.uint64)
    coff[2], coff[3] = coff[3], coff[2] - 1
    with pytest.raises(gpu.PhantGpuError) as e:
        ctx.read_state(r["n_nodes"], r["nodes"], r["node_off"], na, r["account_keys32"], r["roots32"], na, n_codes=len(r["codes"]), codes=cdata,
                       code_off=coff, account_status=np.zeros(na, np.uint8))
    assert e.value.code == -1
    st = ctx.stats()
    assert st["launches"] == 0 and st["h2d_bytes"] == 0


def test_launch_count_does_not_depend_on_the_number_of_reads(ctx, fixture):
    r = fixture
    counts = []
    for n in (10, 100_000):
        ia = np.arange(n) % (r["account_keys32"].size // 32)
        iss = np.arange(n) % (r["slot_keys32"].size // 32)
        akeys = np.ascontiguousarray(r["account_keys32"].reshape(-1, 32)[ia])
        roots = np.ascontiguousarray(r["roots32"].reshape(-1, 32)[ia])
        # slot j keeps its account: the account list is tiled, so slot_account maps into the first copy
        ctx.reset_stats()
        got = gpu_read(ctx, r["nodes"], r["node_off"], roots, akeys, np.ascontiguousarray(r["slot_keys32"].reshape(-1, 32)[iss]),
                       np.minimum(r["slot_account"][iss], n - 1).astype(np.uint32), r["codes"], want=("account_status", "slot_status"))
        counts.append(ctx.stats()["launches"])
        assert (got["account_status"] != 0x77).all() and (got["slot_status"] != 0x77).all()
    assert counts[0] == counts[1] and counts[0] > 0, counts


# ---- 5. the C5 block witnesses ------------------------------------------------------------------------------------------------
def c5_reads(w):
    """the node arena of synth_blocks as one node set; per transaction the two accounts (sender A, contract B) under the
    block's state root and B's two slots"""
    n_tx = w["n_proofs"] // 4
    keys = w["keys32"].view(n_tx, 4, 32)
    roots = w["roots32"].view(n_tx, 4, 32)
    akeys = keys[:, :2].reshape(-1).contiguous()
    aroots = roots[:, :2].reshape(-1).contiguous()
    skeys = keys[:, 2:].reshape(-1).contiguous()
    import torch
    sacc = (2 * torch.arange(2 * n_tx, device=akeys.device, dtype=torch.int64).div(2, rounding_mode="floor") + 1).to(torch.int32)
    return n_tx, akeys, aroots, skeys, sacc


def c5_call(ctx, w, extra_out=()):
    import torch
    from phant_b200 import gpu
    n_tx, akeys, aroots, skeys, sacc = c5_reads(w)
    na, ns = 2 * n_tx, 2 * n_tx
    dev = akeys.device
    out = dict(account_status=torch.zeros(na, dtype=torch.uint8, device=dev), nonce=torch.zeros(na, dtype=torch.int64, device=dev),
               balance32=torch.zeros(na * 32, dtype=torch.uint8, device=dev), storage_root32=torch.zeros(na * 32, dtype=torch.uint8, device=dev),
               code_hash32=torch.zeros(na * 32, dtype=torch.uint8, device=dev), code_index=torch.zeros(na, dtype=torch.int32, device=dev),
               slot_status=torch.zeros(ns, dtype=torch.uint8, device=dev), slot_vals32=torch.zeros(ns * 32, dtype=torch.uint8, device=dev))
    torch.cuda.synchronize()
    ctx.set_flags(gpu.FLAG_DEVICE_PTRS)
    try:
        ctx.read_state(w["n_nodes"], w["nodes"], w["node_off"], na, akeys, aroots, na, ns, skeys, sacc, nodes_bytes=w["n_bytes"], **out)
        ctx.synchronize()
    finally:
        ctx.set_flags(0)
    return (akeys, aroots, skeys, sacc), out


def test_device_built_block_witnesses_vs_oracle(ctx, oracle):
    import torch
    from phant_b200 import synth_blocks
    first, nb, txs = 30, 12, 40
    w = synth_blocks.synth_blocks(ctx, "cuda", first, nb, txs=txs)
    (akeys, aroots, skeys, sacc), out = c5_call(ctx, w)
    h = lambda t: t.cpu().numpy()
    want = read_state(oracle, h(w["nodes"]), h(w["node_off"]).view(np.uint64), h(aroots), h(akeys), h(skeys), h(sacc).view(np.uint32))
    got = {k: h(v) for k, v in out.items()}
    for k in FIELDS:
        assert (got[k].view(np.uint8).reshape(-1) == np.ascontiguousarray(want[k]).view(np.uint8).reshape(-1)).all(), k
    bad = np.nonzero(got["account_status"] != 1)[0]
    assert bad.tolist() == [(37 - first) * 2 * txs] and got["account_status"][bad[0]] == 3
    assert (got["slot_status"] == 1).all()


def test_full_size_block_witnesses(ctx):
    """1000 blocks x 300 transactions: 600k account reads and 600k slot reads in one call"""
    import torch
    from phant_b200 import synth_blocks
    nb, txs = 1000, 300
    w = synth_blocks.synth_blocks(ctx, "cuda", 0, nb, txs=txs)
    (akeys, aroots, skeys, sacc), out = c5_call(ctx, w)
    n_tx = nb * txs
    st = out["account_status"].cpu()
    expect = torch.ones(2 * n_tx, dtype=torch.uint8)
    bad = torch.arange(nb)[torch.arange(nb) % 100 == 37] * 2 * txs
    expect[bad] = 3
    assert torch.equal(st, expect)
    assert bool((out["slot_status"] == 1).all())
    # each slot value = the 32 bytes after 0xa0 in its storage leaf (the last node of its proof)
    pf, ni, off = w["proof_first"], w["node_index"], w["node_off"]
    slot_proofs = (torch.arange(n_tx, device=pf.device).unsqueeze(1) * 4 + torch.tensor([2, 3], device=pf.device)).reshape(-1)
    leaf = ni[pf[slot_proofs + 1] - 1]
    start = off[leaf] + 35
    assert bool((w["nodes"][start - 1] == 0xA0).all())
    vals = w["nodes"][start.unsqueeze(1) + torch.arange(32, device=start.device)]
    assert torch.equal(vals.reshape(-1), out["slot_vals32"])
    # each contract's storage root = the generator's storage root of its slots
    sroot = w["roots32"].view(n_tx, 4, 32)[:, 2]
    assert torch.equal(out["storage_root32"].view(n_tx, 2, 32)[:, 1], sroot)


# ---- the Python host mirror ----------------------------------------------------------------------------------------------------
def test_read_payload_witness_loads_a_statedb(ctx, oracle, golden):
    """host.read_payload_witness on a witness blob per fixture table: the StateDB it fills has the fixture's state root"""
    from phant_b200.host import encode_witness, read_payload_witness
    g = golden("fixture_states.json.gz")
    root_of = fixture_roots(g)
    from helpers import rlp_int_be, secure_account_items
    done = 0
    for tab, accounts in sorted(g["tables"].items()):
        if not accounts or not any(a["storage"] for a in accounts):
            continue
        trie = oracle.trie(secure_account_items(oracle.keccak256, oracle.mptize, accounts))
        nodes, slots = {}, []
        absent = bytes(range(20))
        for a in accounts + [dict(address=absent.hex(), storage={})]:
            for nd in trie.prove(oracle.keccak256(bytes.fromhex(a["address"]))):
                nodes[nd] = 1
            st = sorted((oracle.keccak256(bytes.fromhex(k)), rlp_int_be(bytes.fromhex(v))) for k, v in a["storage"].items() if int(v, 16))
            strie = oracle.trie(st) if st else None
            for k, v in a["storage"].items():
                slots.append((bytes.fromhex(a["address"]), int(k, 16)))
                if strie is not None:
                    for nd in strie.prove(oracle.keccak256(bytes.fromhex(k))):
                        nodes[nd] = 1
        codes = [bytes.fromhex(a["code"]) for a in accounts if a["code"]]
        blob = encode_witness([], codes, list(nodes))
        pre = read_payload_witness(ctx, bytes.fromhex(root_of[tab]), blob, [bytes.fromhex(a["address"]) for a in accounts] + [absent], slots)
        assert pre.complete and pre.account_status[absent] == 2 and absent not in pre.accounts
        for a in accounts:
            s = pre.accounts[bytes.fromhex(a["address"])]
            assert s.nonce == a["nonce"] and s.balance == int(a["balance"], 16) and s.code == bytes.fromhex(a["code"])
            assert s.storage == {int(k, 16): int(v, 16) for k, v in a["storage"].items() if int(v, 16)}
        assert pre.statedb().root(ctx).hex() == root_of[tab], tab
        # without its codes the witness is incomplete
        if codes:
            pre = read_payload_witness(ctx, bytes.fromhex(root_of[tab]), encode_witness([], [], list(nodes)), [], slots)
            assert not pre.complete and pre.missing_code
        done += 1
    assert done >= 10
