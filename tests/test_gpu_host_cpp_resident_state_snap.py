"""snap's GetAccountRange / GetStorageRanges answers from the resident world state in C++ (host/phant_host.hpp:
ResidentStateTrie::snapAccountRange / snapStorageRanges) over the C ABI: compiles and links on the CPU; on the GPU
host/resident_state_snap_test.cpp syncs every fixture's pre-state through them with small budgets, checks every answer with
G (snap::verifySnapAccountRange / verifySnapStorageRanges) and compares the accounts and slots it gathered with the state."""
import os
import subprocess

import pytest

from test_gpu_host_cpp_resident_state_witness import write_cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(out_dir):
    from phant_b200 import gpu
    lib = os.path.dirname(gpu.LIB_PATH)
    exe = os.path.join(str(out_dir), "resident_state_snap_test")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "host", "resident_state_snap_test.cpp"),
                    f"-L{lib}", "-lphantgpu", f"-Wl,-rpath,{lib}"], check=True)
    return exe


def test_resident_state_snap_mirror_compiles_and_links(tmp_path):
    assert os.path.exists(build(tmp_path))


@pytest.mark.gpu
def test_fixture_sync_through_the_cpp_mirror(golden, tmp_path):
    exe = build(tmp_path)
    cases = str(tmp_path / "cases.txt")
    n = write_cases(golden("fixture_states.json.gz"), cases)
    assert n == 84
    r = subprocess.run([exe, cases], capture_output=True, text=True)
    assert r.returncode == 0 and "ALL OK" in r.stdout and f"{n} cases" in r.stdout, r.stdout + r.stderr
