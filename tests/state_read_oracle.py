"""The rules of entry point P (pre-state reads, DESIGN.md "P: pre-state reads") stated on the CPU for the tests: the oracle's
bag walk (oracle_verify_bag, sorted-digest lookup) for the account and slot walks, and its own RLP decode of the account body
and the slot value, written without looking at phant_b200/csrc/state_read.cuh.  Also builds the fixture node sets the CPU and
GPU tests share.  TEST INFRASTRUCTURE: the product never imports this."""
import numpy as np

import oracle_lib
from helpers import rlp_int_be, secure_account_items

CODE_EMPTY = 0xFFFFFFFF
CODE_MISSING = 0xFFFFFFFE
EMPTY_CODE_HASH = bytes.fromhex("c5d2460186f7233c927e7db2dcc703c0e500b653ca82273b7bfad8045d85a470")


def _item(b, pos, end):
    """one canonical RLP item at b[pos:end] -> (is_list, payload_start, payload_end) or None"""
    if pos >= end:
        return None
    t = b[pos]
    if t < 0x80:
        return False, pos, pos + 1
    is_list = t >= 0xC0
    t -= 0xC0 if is_list else 0x80
    if t < 56:
        start, n = pos + 1, t
        if not is_list and n == 1 and (start >= end or b[start] < 0x80):
            return None
    else:
        ll = t - 55
        if ll > 4 or pos + 1 + ll > end or b[pos + 1] == 0:
            return None
        n = int.from_bytes(b[pos + 1:pos + 1 + ll], "big")
        if n < 56:
            return None
        start = pos + 1 + ll
    if start + n > end:
        return None
    return is_list, start, start + n


def decode_account(body):
    """proven account value -> (nonce, balance bytes, storage root, code hash) or None when it breaks a rule"""
    b = bytes(body)
    top = _item(b, 0, len(b))
    if top is None or not top[0] or top[2] != len(b):
        return None
    fields, pos = [], top[1]
    while pos < top[2]:
        it = _item(b, pos, top[2])
        if it is None or it[0]:
            return None
        fields.append(b[it[1]:it[2]])
        pos = it[2]
    if len(fields) != 4:
        return None
    nonce, bal, root, code = fields
    if len(nonce) > 8 or nonce[:1] == b"\x00" or len(bal) > 32 or bal[:1] == b"\x00" or len(root) != 32 or len(code) != 32:
        return None
    return int.from_bytes(nonce, "big"), bal, root, code


def decode_slot(payload):
    """proven slot value -> the value bytes (1..32, first byte non-zero) or None"""
    b = bytes(payload)
    it = _item(b, 0, len(b))
    if it is None or it[0] or it[2] != len(b):
        return None
    v = b[it[1]:it[2]]
    return v if 1 <= len(v) <= 32 and v[0] != 0 else None


def read_state(oracle, nodes, node_off, roots32, account_keys32, slot_keys32=None, slot_account=None, codes=()):
    """-> dict of numpy arrays, the outputs of phant_gpu_read_state (roots32: 1 or n_accounts roots)"""
    na = account_keys32.size // 32
    ns = 0 if slot_keys32 is None else slot_keys32.size // 32
    out = dict(account_status=np.zeros(na, np.uint8), nonce=np.zeros(na, np.uint64), balance32=np.zeros((na, 32), np.uint8),
               storage_root32=np.zeros((na, 32), np.uint8), code_hash32=np.zeros((na, 32), np.uint8),
               code_index=np.full(na, CODE_EMPTY, np.uint32), slot_status=np.zeros(ns, np.uint8), slot_vals32=np.zeros((ns, 32), np.uint8))
    nodes = np.ascontiguousarray(nodes)
    by_hash = {}
    for i, c in enumerate(codes):
        by_hash.setdefault(oracle.keccak256(bytes(c)), i)
    if na:
        st, vo, vl = oracle.verify_bag(nodes, node_off, np.ascontiguousarray(account_keys32), np.ascontiguousarray(roots32), threads=4)
        for i in range(na):
            s = int(st[i])
            if s == 1:
                acc = decode_account(nodes[int(vo[i]):int(vo[i]) + int(vl[i])].tobytes())
                if acc is None:
                    s = 0
                else:
                    nonce, bal, root, code = acc
                    out["nonce"][i] = nonce
                    out["balance32"][i] = np.frombuffer(bal.rjust(32, b"\x00"), np.uint8)
                    out["storage_root32"][i] = np.frombuffer(root, np.uint8)
                    out["code_hash32"][i] = np.frombuffer(code, np.uint8)
                    if code != EMPTY_CODE_HASH:
                        out["code_index"][i] = by_hash.get(code, CODE_MISSING)
            out["account_status"][i] = s
    if ns:
        acc = np.asarray(slot_account, np.int64)
        ok = acc < na
        walk = np.nonzero(ok)[0]
        walk = walk[out["account_status"][acc[walk]] == 1]
        out["slot_status"][:] = 0
        out["slot_status"][ok] = out["account_status"][acc[ok]]
        if walk.size:
            keys = np.ascontiguousarray(slot_keys32.reshape(-1, 32)[walk])
            roots = np.ascontiguousarray(out["storage_root32"][acc[walk]])
            st, vo, vl = oracle.verify_bag(nodes, node_off, keys, roots, threads=4)
            for j, i in enumerate(walk):
                s = int(st[j])
                if s == 1:
                    v = decode_slot(nodes[int(vo[j]):int(vo[j]) + int(vl[j])].tobytes())
                    if v is None:
                        s = 0
                    else:
                        out["slot_vals32"][i] = np.frombuffer(v.rjust(32, b"\x00"), np.uint8)
                out["slot_status"][i] = s
    return out


# ---- the fixture node sets (tests/golden/fixture_states.json.gz) ------------------------------------------------------------
def fixture_roots(g):
    """table name -> the state root a fixture header pins it to"""
    root_of = {}
    for t in g["tests"]:
        for tab, root in ((t["pre"], t["pre_root"]), (t["post"], t["post_root"])):
            assert root_of.setdefault(tab, root) == root
    return root_of


def fixture_reads(oracle, g, seed=7):
    """every account and non-zero slot of all fixture tables, plus absent accounts and absent slots (under present and absent
    accounts), with the node set that proves them and the codes of every table plus junk.  -> dict with the call's inputs and,
    per read, the expectation taken from the fixture table itself: account_want[i] = (table, account) or None (absent),
    slot_want[i] = (status, 32-byte value, slot number bytes or None)"""
    rng = np.random.default_rng(seed)
    root_of = fixture_roots(g)
    nodes, codes = {}, {}
    acc_keys, acc_roots, acc_want, slot_keys, slot_acc, slot_want = [], [], [], [], [], []
    for tab, accounts in sorted(g["tables"].items()):
        froot = bytes.fromhex(root_of[tab])
        trie = oracle.trie(secure_account_items(oracle.keccak256, oracle.mptize, accounts)) if accounts else None

        def add_account(key, want):
            if trie is not None:
                for nd in trie.prove(key):
                    nodes[nd] = 1
            acc_keys.append(key)
            acc_roots.append(froot)
            acc_want.append(want)
            return len(acc_keys) - 1

        for a in accounts:
            ai = add_account(oracle.keccak256(bytes.fromhex(a["address"])), (tab, a))
            if a["code"]:
                codes[bytes.fromhex(a["code"])] = 1
            st = sorted((oracle.keccak256(bytes.fromhex(k)), rlp_int_be(bytes.fromhex(v)), bytes.fromhex(v), bytes.fromhex(k))
                        for k, v in a["storage"].items() if int(v, 16) != 0)
            strie = oracle.trie([(k, v) for k, v, _, _ in st]) if st else None
            for k, _, raw, pre in st:
                for nd in strie.prove(k):
                    nodes[nd] = 1
                slot_keys.append(k); slot_acc.append(ai); slot_want.append((1, raw.lstrip(b"\x00").rjust(32, b"\x00"), pre))
            absent = oracle.keccak256(b"absent slot" + a["address"].encode())
            if strie is not None:
                for nd in strie.prove(absent):
                    nodes[nd] = 1
            slot_keys.append(absent); slot_acc.append(ai); slot_want.append((2, bytes(32), None))
        for _ in range(2):
            k = rng.integers(0, 256, 32, dtype=np.uint8).tobytes()
            ai = add_account(k, None)
            slot_keys.append(oracle.keccak256(k)); slot_acc.append(ai); slot_want.append((2, bytes(32), None))
    code_list = list(codes) + [b"junk code %d" % i for i in range(5)] + [b""]
    rng.shuffle(code_list)
    node_list = list(nodes)
    data, off = oracle_lib.csr(node_list, np.uint64)
    return dict(nodes=np.concatenate([data, np.zeros(64, np.uint8)]), node_off=off, n_nodes=len(node_list), node_list=node_list,
                codes=code_list, account_keys32=np.frombuffer(b"".join(acc_keys), np.uint8).copy(),
                roots32=np.frombuffer(b"".join(acc_roots), np.uint8).copy(), account_want=acc_want,
                slot_keys32=np.frombuffer(b"".join(slot_keys), np.uint8).copy(), slot_account=np.array(slot_acc, np.uint32), slot_want=slot_want)


def check_against_fixture(r, got, codes):
    """assert that the read values `got` (dict as read_state returns) are what the fixture tables say"""
    for i, want in enumerate(r["account_want"]):
        if want is None:
            assert got["account_status"][i] == 2 and got["nonce"][i] == 0 and not got["balance32"][i].any(), i
            assert got["code_index"][i] == CODE_EMPTY
            continue
        _, a = want
        assert got["account_status"][i] == 1, i
        assert int(got["nonce"][i]) == a["nonce"]
        assert got["balance32"][i].tobytes() == bytes.fromhex(a["balance"]).rjust(32, b"\x00")
        ci = int(got["code_index"][i])
        if a["code"]:
            assert ci < len(codes) and bytes(codes[ci]) == bytes.fromhex(a["code"]), i
        else:
            assert ci == CODE_EMPTY, i
    for i, (st, val, _) in enumerate(r["slot_want"]):
        assert got["slot_status"][i] == st, (i, got["slot_status"][i], st)
        assert got["slot_vals32"][i].tobytes() == val, i
