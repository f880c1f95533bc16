"""Undo through the C++ resident state (host/phant_host.hpp: state::ResidentStateTrie::setJournal / revert): compiles and links
on the CPU; on the GPU host/resident_state_revert_test.cpp applies blocks against StateDB::root(), reverts and applies again."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build(out_dir):
    from phant_b200 import gpu
    lib = os.path.dirname(gpu.LIB_PATH)
    exe = os.path.join(str(out_dir), "resident_state_revert_test")
    subprocess.run(["g++", "-std=c++17", "-O1", "-Wall", "-Werror", "-o", exe, os.path.join(ROOT, "host", "resident_state_revert_test.cpp"),
                    f"-L{lib}", "-lphantgpu", f"-Wl,-rpath,{lib}"], check=True)
    return exe


def test_revert_mirror_compiles_and_links(tmp_path):
    assert os.path.exists(build(tmp_path))


@pytest.mark.gpu
def test_invalid_blocks_and_a_reorg_through_the_cpp_mirror(tmp_path):
    r = subprocess.run([build(tmp_path)], capture_output=True, text=True)
    assert r.returncode == 0 and "ALL OK" in r.stdout, r.stdout + r.stderr
