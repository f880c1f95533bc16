"""The CPU statement of pre-state reads (tests/state_read_oracle.py) against the fixture tables, without a GPU: every account
and every non-zero slot of all 91 tables read back from a node set under the root the fixture headers pin, absent reads
proven absent, codes found by hash."""
import numpy as np

import oracle_lib
from state_read_oracle import CODE_EMPTY, CODE_MISSING, check_against_fixture, decode_account, decode_slot, fixture_reads, read_state


def test_fixture_tables_read_back(oracle, golden):
    g = golden("fixture_states.json.gz")
    r = fixture_reads(oracle, g)
    assert len(g["tables"]) == 91
    got = read_state(oracle, r["nodes"], r["node_off"], r["roots32"], r["account_keys32"], r["slot_keys32"], r["slot_account"], r["codes"])
    check_against_fixture(r, got, r["codes"])
    assert (got["account_status"] == 1).sum() >= 1100 and (got["slot_status"] == 1).sum() >= 70


def test_oracle_rules_on_crafted_values(oracle):
    """the account and slot rules decide the status, and an incomplete or rejected account passes its status to its slots"""
    from helpers import rlp_list, rlp_str
    good = rlp_list([b"\x05", rlp_str(b"\x01\x00"), rlp_str(bytes(range(32))), rlp_str(bytes(32))])
    assert decode_account(good) == (5, b"\x01\x00", bytes(range(32)), bytes(32))
    assert decode_account(rlp_list([b"\x00", rlp_str(b"\x01"), rlp_str(bytes(32)), rlp_str(bytes(32))])) is None  # nonce 0x00
    assert decode_account(good + b"\x00") is None
    assert decode_slot(b"\x05") == b"\x05" and decode_slot(b"\x80") is None and decode_slot(b"\x00") is None
    assert decode_slot(rlp_str(b"\x00\x01")) is None and decode_slot(rlp_str(bytes([1]) * 33)) is None
    # one account with a storage trie; its code is missing from the codes
    skey = oracle.keccak256(b"slot")
    strie = oracle.trie([(skey, b"\x2a")])
    akey = oracle.keccak256(b"addr")
    body = rlp_list([b"\x01", rlp_str(b"\x02"), rlp_str(strie.root()), rlp_str(oracle.keccak256(b"code"))])
    atrie = oracle.trie([(akey, body)])
    nodes = list({nd: 1 for nd in atrie.prove(akey) + strie.prove(skey)})
    data, off = oracle_lib.csr(nodes, np.uint64)
    keys = np.frombuffer(akey + oracle.keccak256(b"other"), np.uint8).copy()
    got = read_state(oracle, data, off, np.frombuffer(atrie.root(), np.uint8).copy(), keys,
                     np.frombuffer(skey + skey, np.uint8).copy(), np.array([0, 1], np.uint32), codes=[b"other code"])
    assert got["account_status"].tolist() == [1, 2] and got["code_index"].tolist() == [CODE_MISSING, CODE_EMPTY]
    assert got["slot_status"].tolist() == [1, 2] and got["slot_vals32"][0, 31] == 0x2A
    # the storage node removed: the slot lacks a node, the account is still present
    data, off = oracle_lib.csr(atrie.prove(akey), np.uint64)
    got = read_state(oracle, data, off, np.frombuffer(atrie.root(), np.uint8).copy(), keys[:32].copy(), np.frombuffer(skey, np.uint8).copy(),
                     np.array([0], np.uint32))
    assert got["account_status"].tolist() == [1] and got["slot_status"].tolist() == [3]
