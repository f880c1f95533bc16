"""The proof walk's decoding rules (R2-R4) on malformed nodes whose hashes still match (tests/walk_corpus.py), on the CPU:
the oracle, the Python statement and the status each case prescribes agree; the device sources compiled as host code --
the two-kernel walk (walk_one.cuh, summary off / staged / direct, plain and deduplicated chains, node sets) and the fused
hash-and-walk lane (verify_fused.cuh, batch order and regrouped) -- equal the oracle; and a coverage build shows that the
corpus executes every return of the decoding functions.  T's node decoder, which shares rlp_item, is checked on every
corpus node too."""
import _ctypes
import ctypes as C
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import oracle_lib
import walk_corpus as wc
from helpers import py_verify
from test_fused_header_host import all_perms, assert_same, hostfused, proof_order, run_fused  # noqa: F401  (fixture)
from test_oracle_proofs import batch_of
from test_transition_header_host import device_decode, lib as transition_lib  # noqa: F401  (fixture)
from test_walk_header_host import _p, digests_of, hostwalk, run_chain  # noqa: F401  (fixture)
from transition_oracle import decode

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), "phant_b200", "csrc")


@pytest.fixture(scope="module")
def corpus(oracle):
    return wc.build(oracle.keccak256)


@pytest.fixture(scope="module")
def batch(corpus):
    return batch_of([c.proof() for c in corpus])


@pytest.fixture(scope="module")
def want(oracle, batch):
    return oracle.verify_proofs(*batch, threads=4)


def test_prescribed_status(oracle, corpus, batch, want):
    """oracle == Python statement == the status the rules prescribe, and the value slice is the prescribed value"""
    nodes = batch[0]
    _, status, voff, vlen = want
    named = 0
    for i, c in enumerate(corpus):
        st, val = py_verify(oracle.keccak256, *c.proof())
        assert st == status[i], (c.name, st, int(status[i]))
        if c.status is not None:
            named += 1
            assert st == c.status, (c.name, st, c.status)
        if st == 1:
            got = nodes[int(voff[i]):int(voff[i]) + int(vlen[i])].tobytes()
            assert got == val, c.name
            if c.status is not None:
                assert got == c.value, c.name
    assert named > 3000 and set(status.tolist()) == {0, 1, 2}
    # the random damage reaches every verdict too, not only R1 rejects
    dmg = np.array([c.status is None for c in corpus])
    assert set(status[dmg].tolist()) == {0, 1, 2}


def check_walk(got, want, what):
    status, voff, vlen = got
    bad = np.nonzero(status != want[1])[0]
    assert bad.size == 0, (what, bad[:10], status[bad[:10]], want[1][bad[:10]])
    ok = status == 1
    assert (voff[ok] == want[2][ok]).all() and (vlen[ok] == want[3][ok]).all(), what


def test_host_walk_chains(hostwalk, oracle, corpus, batch, want):  # noqa: F811
    """walk_one.cuh as host code, chain form: summary off, as the staged kernel leaves it, as the direct kernel leaves it;
    and the same proofs deduplicated (chains of node indices, shared nodes)"""
    for use_summary in (0, 1, 2):
        check_walk(run_chain(hostwalk, oracle, *batch, use_summary), want, use_summary)
    flat = [nd for c in corpus for nd in c.nodes]
    uniq = list({nd: 1 for nd in flat})
    assert len(uniq) < len(flat)
    where = {nd: j for j, nd in enumerate(uniq)}
    unodes, uoff = oracle_lib.csr(uniq, np.uint64)
    index = np.array([where[nd] for nd in flat], np.uint64)
    _, _, first, keys, roots = batch
    want_d = oracle.verify_proofs(unodes, uoff, first, keys, roots, threads=4, node_index=index)
    assert (want_d[1] == want[1]).all()
    for use_summary in (0, 1):
        check_walk(run_chain(hostwalk, oracle, unodes, uoff, first, keys, roots, use_summary, node_index=index), want_d, ("dedup", use_summary))


def bag_of(corpus, leave_out=False):
    """every node of every case in one node set (each case has its own root); leave_out drops each case's node under test"""
    drop = {c.nodes[c.target] for c in corpus if leave_out and c.target is not None and c.name != "spacer"}
    return list({nd: 1 for c in corpus for nd in c.nodes if nd not in drop})


def run_bag(lib, oracle, bag, keys, roots, use_summary):
    bnodes, boff = oracle_lib.csr(bag, np.uint64)
    n = keys.size // 32
    st, vo, vl = np.full(n, 9, np.uint8), np.zeros(n, np.uint64), np.zeros(n, np.uint32)
    padded = np.concatenate([bnodes, np.zeros(64, np.uint8)])
    lib.hostwalk_bag(_p(padded), _p(boff), C.c_uint64(len(bag)), C.c_uint64(n), _p(keys), _p(roots), C.c_uint64(n),
                     _p(digests_of(oracle, bnodes, boff)), C.c_int(use_summary), _p(st), _p(vo), _p(vl))
    return bnodes, boff, (st, vo, vl)


def test_host_walk_bags(hostwalk, oracle, corpus, batch):  # noqa: F811
    """the same cases as node sets: complete, and with each case's malformed node left out (ST_MISSING)"""
    _, _, _, keys, roots = batch
    for leave_out in (False, True):
        bag = bag_of(corpus, leave_out)
        bnodes, boff, got = run_bag(hostwalk, oracle, bag, keys, roots, 1)
        want_bag = oracle.verify_bag(bnodes, boff, keys, roots, threads=4)
        assert (got[0] == want_bag[0]).all(), (leave_out, np.nonzero(got[0] != want_bag[0])[0][:10])
        ok = got[0] == 1
        assert (got[1][ok] == want_bag[1][ok]).all() and (got[2][ok] == want_bag[2][ok]).all()
        if leave_out:
            reach = np.array([c.target is not None and c.name != "spacer" for c in corpus])
            assert (want_bag[0][reach] == wc.MISSING).all()
        else:  # a hash reference at a chain's end names no node of the set: missing, not rejected, in a node set
            assert set(want_bag[0].tolist()) == {0, 1, 2, 3}


def test_host_fused(hostfused, oracle, batch, want):  # noqa: F811
    """verify_fused.cuh as host code: batch order and regrouped order, and the Keccak work it reports"""
    got = run_fused(hostfused, *batch)
    assert_same(got, want)
    assert int(got[3][2]) == all_perms(batch[1])
    again = run_fused(hostfused, *batch, proof_order(batch[2]))
    for a, b in zip(again[:3], got[:3]):
        assert (a == b).all()


def test_solo_at_buffer_start(hostwalk, hostfused, oracle, corpus):  # noqa: F811
    """each depth-0 case alone, so its node starts the node buffer: leaves under 48 bytes into it compare their path
    nibble by nibble instead of with the wide load; every start residue is covered by the corpus itself"""
    solo = [c for c in corpus if "/d0/" in c.name]
    assert len(solo) > 300
    for c in solo:
        b = batch_of([c.proof()])
        w = oracle.verify_proofs(*b)
        assert int(w[1][0]) == c.status, c.name
        check_walk(run_chain(hostwalk, oracle, *b, 1), w, c.name)
        assert_same(run_fused(hostfused, *b), w)


def test_transition_decoder(transition_lib, corpus):  # noqa: F811
    """T's host-compiled node decoder (tn_decode, which shares rlp_item) against transition_oracle.decode on every node"""
    seen = set()
    for c in corpus:
        for nd in c.nodes:
            if nd in seen or len(nd) > 5000:
                continue
            seen.add(nd)
            assert device_decode(transition_lib, nd) == decode(nd), (c.name, nd[:16].hex())
    assert len(seen) > 5000


# ---- coverage gate ---------------------------------------------------------------------------------------------------
# Returns the corpus may leave unexecuted, with the reason.  Keyed by (file, function, the line's text stripped).
ALLOWED_UNREACHED = {
    ("walk_one.cuh", "walk_one", "if (l > 0xffffffffull) return ST_REJECT;"):
        "a node over 4 GiB: no test can hold one",
}
GATED = {"walk_one.cuh": ("rlp_item", "walk_node", "walk_one"), "node_summary.cuh": ("summarize_node",), "verify_fused.cuh": ("fused_step",)}


def function_lines(src, name):
    """1-based line range of the function `name` in src: its definition (the `__device__` line that names it, at column 0)
    to the closing brace at column 0.  Exactly one definition must match."""
    lines = src.split("\n")
    starts = [i for i, ln in enumerate(lines) if re.match(r"__device__\b.*\b%s\(" % name, ln)]
    assert len(starts) == 1, (name, starts)
    end = next(i for i in range(starts[0], len(lines)) if lines[i].startswith("}"))
    return starts[0] + 1, end + 1


def return_lines(src, name):
    """{line number: stripped text} of every line of function `name` with a `return` outside a comment"""
    lines = src.split("\n")
    a, b = function_lines(src, name)
    return {n: lines[n - 1].strip() for n in range(a, b + 1) if re.search(r"\breturn\b", lines[n - 1].split("//")[0])}


def fully_run_lines(gcov_text):
    """line numbers gcov shows executed with every block on them executed (count not '#####'/'=====', no '*' suffix)"""
    out = set()
    for ln in gcov_text.split("\n"):
        m = re.match(r"\s*([^:]+):\s*(\d+):", ln)
        if not m or int(m.group(2)) == 0:
            continue
        c = m.group(1).strip()
        if c != "-" and not c.startswith(("#####", "=====")) and not c.endswith("*"):
            out.add(int(m.group(2)))
    return out


def test_gate_finds_every_gated_function():
    """the gate looks at each function's own body: a definition, not a comment naming it, and at least one return"""
    for hdr, funcs in GATED.items():
        src = open(os.path.join(CSRC, hdr)).read()
        for fn in funcs:
            a, _ = function_lines(src, fn)
            assert src.split("\n")[a - 1].startswith("__device__"), (hdr, fn)
            assert return_lines(src, fn), (hdr, fn)


@pytest.mark.skipif(shutil.which("gcov") is None, reason="gcov is not installed")
def test_coverage_gate(oracle, corpus, batch, want, tmp_path):
    """build walk_host.cpp and fused_host.cpp again with --coverage -O0, run the whole corpus through them and require
    every return of rlp_item, walk_node, walk_one, summarize_node and fused_step to have run (whole line, every block on it)"""
    libs = {}
    for name in ("walk_host", "fused_host"):
        d = tmp_path / name
        d.mkdir()
        obj = d / (name + ".o")
        subprocess.run(["g++", "-O0", "--coverage", "-std=c++17", "-fPIC", "-Wno-unknown-pragmas", "-c", "-o", str(obj),
                        os.path.join(HERE, "hostcheck", name + ".cpp")], check=True, cwd=d)
        so = d / ("lib" + name + ".so")
        subprocess.run(["g++", "--coverage", "-shared", "-o", str(so), str(obj)], check=True, cwd=d)
        libs[name] = (d, obj, C.CDLL(str(so)))
    walk, fused = libs["walk_host"][2], libs["fused_host"][2]
    for use_summary in (0, 1, 2):
        check_walk(run_chain(walk, oracle, *batch, use_summary), want, use_summary)
    _, _, _, keys, roots = batch
    for leave_out in (False, True):
        run_bag(walk, oracle, bag_of(corpus, leave_out), keys, roots, 1)
    assert_same(run_fused(fused, *batch), want)
    for c in corpus:
        if "/d0/" in c.name:
            b = batch_of([c.proof()])
            run_chain(walk, oracle, *b, 1)
            run_fused(fused, *b)
    # a return counts as reached when either build ran all of its line (walk_node's summary fast path, for one, is only
    # taken in the two-kernel walk: the fused lane reads a simple branch's child from its slot instead)
    run = {hdr: set() for hdr in GATED}
    seen = {hdr: [] for hdr in GATED}
    for name, (d, obj, lib) in libs.items():
        _ctypes.dlclose(lib._handle)  # unloading the library writes its .gcda
        assert os.path.exists(str(obj)[:-2] + ".gcda"), name
        subprocess.run(["gcov", "-o", str(d), os.path.join(HERE, "hostcheck", name + ".cpp")], check=True, cwd=d,
                       stdout=subprocess.DEVNULL)
        for hdr in GATED:
            g = d / (hdr + ".gcov")
            if g.exists():
                seen[hdr].append(name)
                run[hdr] |= fully_run_lines(g.read_text())
    missing = [hdr for hdr, builds in seen.items() if not builds]
    assert not missing, f"no build produced a .gcov for {missing}"
    problems = []
    for hdr, funcs in GATED.items():
        src = open(os.path.join(CSRC, hdr)).read()
        for fn in funcs:
            for n, text in return_lines(src, fn).items():
                if n not in run[hdr] and (hdr, fn, text) not in ALLOWED_UNREACHED:
                    problems.append(f"{hdr}:{n} ({fn}): {text}")
    assert not problems, "returns no corpus case reaches:\n" + "\n".join(problems)
