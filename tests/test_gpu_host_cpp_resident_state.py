"""The C++ resident state (host/phant_host.hpp: state::ResidentStateTrie) over the C ABI: compiles and links on the CPU; on
the GPU host/resident_state_test.cpp sends only each block's changed slots and checks every root against StateDB::root()."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(out_dir):
    from phant_b200 import gpu
    lib = os.path.dirname(gpu.LIB_PATH)
    exe = os.path.join(str(out_dir), "resident_state_test")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "host", "resident_state_test.cpp"),
                    f"-L{lib}", "-lphantgpu", f"-Wl,-rpath,{lib}"], check=True)
    return exe


def test_resident_state_mirror_compiles_and_links(tmp_path):
    assert os.path.exists(build(tmp_path))


@pytest.mark.gpu
def test_incremental_blocks_through_the_cpp_mirror(tmp_path):
    r = subprocess.run([build(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
