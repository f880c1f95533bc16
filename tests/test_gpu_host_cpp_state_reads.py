"""The C++ pre-state factory (host/phant_host.hpp: engine_api::readPreState / stateDBFromWitness) over the C ABI: compiles and
links on the CPU; on the GPU host/state_read_test.cpp fills a StateDB from a witness per fixture table and checks its root."""
import os
import subprocess

import pytest

from helpers import rlp_int_be, secure_account_items
from state_read_oracle import fixture_roots

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(out_dir):
    from phant_b200 import gpu
    lib = os.path.dirname(gpu.LIB_PATH)
    exe = os.path.join(str(out_dir), "state_read_test")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "host", "state_read_test.cpp"), f"-L{lib}",
                    "-lphantgpu", f"-Wl,-rpath,{lib}"], check=True)
    return exe


def test_state_read_mirror_compiles_and_links(tmp_path):
    assert os.path.exists(build(tmp_path))


def write_cases(oracle, g, path):
    """one case per non-empty fixture table: the node set proving every account, every stored slot, an absent account and an
    absent slot; the table's codes; the expected root = the table's own root (every non-zero slot is read)"""
    root_of = fixture_roots(g)
    n = 0
    with open(path, "w") as f:
        for tab, accounts in sorted(g["tables"].items()):
            if not accounts:
                continue
            trie = oracle.trie(secure_account_items(oracle.keccak256, oracle.mptize, accounts))
            nodes, lines = {}, []
            absent = bytes([0xAB] * 20)
            for a in accounts + [dict(address=absent.hex(), storage={})]:
                for nd in trie.prove(oracle.keccak256(bytes.fromhex(a["address"]))):
                    nodes[nd] = 1
                st = sorted((oracle.keccak256(bytes.fromhex(k)), rlp_int_be(bytes.fromhex(v))) for k, v in a["storage"].items() if int(v, 16))
                strie = oracle.trie(st) if st else None
                for k in list(a["storage"]) + ["ff" * 32]:
                    slot32 = bytes.fromhex(k).rjust(32, b"\x00")
                    lines.append(f"slot {a['address']} {slot32.hex()}")
                    if strie is not None:
                        for nd in strie.prove(oracle.keccak256(slot32)):
                            nodes[nd] = 1
            # the first account's leaf goes last: the C++ test drops the last node and expects a refusal
            leaf = trie.prove(oracle.keccak256(bytes.fromhex(accounts[0]["address"])))[-1]
            order = [nd for nd in nodes if nd != leaf] + [leaf]
            f.write(f"case {root_of[tab]} {root_of[tab]}\n")
            f.writelines(f"node {nd.hex()}\n" for nd in order)
            f.writelines(f"code {c}\n" for c in sorted({a['code'] for a in accounts if a["code"]}))
            f.writelines(f"addr {a['address']}\n" for a in accounts)
            f.write(f"absent {absent.hex()}\n")
            f.writelines(line + "\n" for line in lines)
            f.write("end\n")
            n += 1
    return n


@pytest.mark.gpu
def test_state_db_from_witness_through_the_cpp_mirror(oracle, golden, tmp_path):
    exe = build(tmp_path)
    cases = str(tmp_path / "cases.txt")
    n = write_cases(oracle, golden("fixture_states.json.gz"), cases)
    assert n >= 50
    r = subprocess.run([exe, cases], capture_output=True, text=True)
    assert r.returncode == 0 and "ALL OK" in r.stdout and f"{n} cases" in r.stdout, r.stdout + r.stderr
