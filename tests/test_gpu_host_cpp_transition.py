"""The C++ transition root (host/phant_host.hpp: engine_api::transitionRoot) over the C ABI: compiles and links on the CPU; on
the GPU host/transition_test.cpp takes every fixture block from its pre-state witness to the header's post root."""
import os
import subprocess

import pytest

from resident_state_model import ZERO32, StateModel, change_diff, hashed_table, load_diff
from transition_oracle import witness

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(out_dir):
    from phant_b200 import gpu
    lib = os.path.dirname(gpu.LIB_PATH)
    exe = os.path.join(str(out_dir), "transition_test")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "host", "transition_test.cpp"), f"-L{lib}",
                    "-lphantgpu", f"-Wl,-rpath,{lib}"], check=True)
    return exe


def test_transition_mirror_compiles_and_links(tmp_path):
    assert os.path.exists(build(tmp_path))


def write_cases(oracle, g, path):
    """one case per fixture: the block's changes by address (accounts created, changed or destroyed; slots written), the
    witness of the pre-state with the account trie's root node last"""
    n = 0
    with open(path, "w") as f:
        for t in g["tests"]:
            pre_t, post_t = g["tables"][t["pre"]], g["tables"][t["post"]]
            pre, post = hashed_table(oracle.keccak256, pre_t), hashed_table(oracle.keccak256, post_t)
            m = StateModel(oracle)
            m.apply(load_diff(pre))
            nodes = witness(oracle, m, change_diff(pre, post))
            root_node = next((nd for nd in nodes if oracle.keccak256(nd).hex() == t["pre_root"]), None)
            if root_node is not None:
                nodes = [nd for nd in nodes if nd != root_node] + [root_node]
            f.write(f"case {t['pre_root']} {t['post_root']}\n")
            f.writelines(f"node {nd.hex()}\n" for nd in nodes)
            by_addr = {a["address"]: a for a in pre_t}
            post_addrs = {a["address"] for a in post_t}
            for a in pre_t:
                if a["address"] not in post_addrs:
                    f.write(f"del {a['address']}\n")
            for a in post_t:
                old = by_addr.get(a["address"])
                norm = lambda st: {bytes.fromhex(k).rjust(32, b"\x00"): bytes.fromhex(v).rjust(32, b"\x00") for k, v in st.items()  # noqa: E731
                                   if int(v, 16)}
                new_s, old_s = norm(a["storage"]), norm(old["storage"]) if old else {}
                writes = {k: v for k, v in new_s.items() if old_s.get(k) != v}
                writes.update({k: ZERO32 for k in old_s if k not in new_s})
                if old and (old["nonce"], int(old["balance"] or "0", 16), old["code"]) == (a["nonce"], int(a["balance"] or "0", 16), a["code"]) \
                        and not writes:
                    continue
                bal = int(a["balance"] or "0", 16).to_bytes(32, "big").hex()
                f.write(f"acct {a['address']} {a['nonce']} {bal} {a['code'] or '-'}\n")
                f.writelines(f"slot {a['address']} {k.hex()} {v.hex()}\n" for k, v in writes.items())
            f.write("end\n")
            n += 1
    return n


@pytest.mark.gpu
def test_fixture_blocks_through_the_cpp_mirror(oracle, golden, tmp_path):
    exe = build(tmp_path)
    cases = str(tmp_path / "cases.txt")
    n = write_cases(oracle, golden("fixture_states.json.gz"), cases)
    assert n == 84
    r = subprocess.run([exe, cases], capture_output=True, text=True)
    assert r.returncode == 0 and "ALL OK" in r.stdout and f"{n} cases" in r.stdout, r.stdout + r.stderr
