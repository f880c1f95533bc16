"""Witnesses from the resident world state in C++ (host/phant_host.hpp: ResidentStateTrie::witness) over the C ABI: compiles
and links on the CPU; on the GPU host/resident_state_witness_test.cpp loads every fixture's pre-state, takes the block's
witness and gets the header's post root from it through engine_api::transitionRoot."""
import os
import subprocess

import pytest

from resident_state_model import ZERO32

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(out_dir):
    from phant_b200 import gpu
    lib = os.path.dirname(gpu.LIB_PATH)
    exe = os.path.join(str(out_dir), "resident_state_witness_test")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "host", "resident_state_witness_test.cpp"),
                    f"-L{lib}", "-lphantgpu", f"-Wl,-rpath,{lib}"], check=True)
    return exe


def test_resident_state_witness_mirror_compiles_and_links(tmp_path):
    assert os.path.exists(build(tmp_path))


def norm(storage):
    return {bytes.fromhex(k).rjust(32, b"\x00"): bytes.fromhex(v).rjust(32, b"\x00") for k, v in storage.items() if int(v, 16)}


def acct_line(kind, a):
    bal = int(a["balance"] or "0", 16).to_bytes(32, "big").hex()
    return f"{kind} {a['address']} {a['nonce']} {bal} {a['code'] or '-'}\n"


def write_cases(g, path):
    """one case per fixture: the pre-state (every account with its storage), then the block's changes by address"""
    n = 0
    with open(path, "w") as f:
        for t in g["tests"]:
            pre_t, post_t = g["tables"][t["pre"]], g["tables"][t["post"]]
            f.write(f"case {t['pre_root']} {t['post_root']}\n")
            for a in pre_t:
                f.write(acct_line("pre", a))
                f.writelines(f"pslot {a['address']} {k.hex()} {v.hex()}\n" for k, v in norm(a["storage"]).items())
            by_addr = {a["address"]: a for a in pre_t}
            post_addrs = {a["address"] for a in post_t}
            f.writelines(f"del {a['address']}\n" for a in pre_t if a["address"] not in post_addrs)
            for a in post_t:
                old = by_addr.get(a["address"])
                new_s, old_s = norm(a["storage"]), norm(old["storage"]) if old else {}
                writes = {k: v for k, v in new_s.items() if old_s.get(k) != v}
                writes.update({k: ZERO32 for k in old_s if k not in new_s})
                if old and (old["nonce"], int(old["balance"] or "0", 16), old["code"]) == (a["nonce"], int(a["balance"] or "0", 16), a["code"]) \
                        and not writes:
                    continue
                f.write(acct_line("acct", a))
                f.writelines(f"slot {a['address']} {k.hex()} {v.hex()}\n" for k, v in writes.items())
            f.write("end\n")
            n += 1
    return n


@pytest.mark.gpu
def test_fixture_blocks_witness_through_the_cpp_mirror(golden, tmp_path):
    exe = build(tmp_path)
    cases = str(tmp_path / "cases.txt")
    n = write_cases(golden("fixture_states.json.gz"), cases)
    assert n == 84
    r = subprocess.run([exe, cases], capture_output=True, text=True)
    assert r.returncode == 0 and "ALL OK" in r.stdout and f"{n} cases" in r.stdout, r.stdout + r.stderr
