"""The device branches of phant_b200/csrc/secp256k1.cuh -- the PTX add.cc / sub.cc chains of add_raw and sub_raw, the asm
rows of mul_wide, fp_reduce's two asm folds, __umul64hi in sc_mul's fold -- on the GPU against Python integers, on the
adversarial corpus of tests/secp_corpus.py (limb patterns, boundary values, pairs landing on p and 2^256, 512-bit inputs
built for fp_reduce's second wrap and sc_mul's fourth round, Jacobian points with z != 1, infinity, p = q and p = -q).

The CPU suite only ever compiles the `#else` branches; the asm is reached here and through the recovery kernel.  The
operations run from tests/devcheck/build/libsecp_devcheck.so (`make -C phant_b200/csrc devcheck`, the library's flags),
one launch per operation, one case per thread; SECP_DEVCHECK_LIB names another build of it."""
import ctypes as C
import os

import numpy as np
import pytest

import secp_corpus

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
LIB = os.environ.get("SECP_DEVCHECK_LIB", os.path.join(HERE, "devcheck", "build", "libsecp_devcheck.so"))


@pytest.fixture(scope="module")
def devcheck():
    if not os.path.exists(LIB):
        pytest.fail(f"{LIB} is missing: build it with `make -C phant_b200/csrc devcheck` (build() does)")
    lib = C.CDLL(LIB)
    lib.secp_check_run.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_uint64]
    in_w, out_w, n_ops = C.c_int(), C.c_int(), C.c_int()
    lib.secp_check_layout(C.byref(in_w), C.byref(out_w), C.byref(n_ops))
    assert (in_w.value, out_w.value, n_ops.value) == (secp_corpus.IN_WORDS, secp_corpus.OUT_WORDS, len(secp_corpus.OPS))
    return lib


@pytest.mark.parametrize("op", secp_corpus.OPS)
def test_device_arithmetic_against_python(devcheck, op):
    """every output equal to Python's value and canonical (below p or n), carry words 0 or 1, mul_wide equal to a * b,
    inverses and square-root candidates equal to pow(), point operations equal to the affine result, every word written"""
    def run(code, inp):
        inp = np.ascontiguousarray(inp)
        out = np.zeros((inp.shape[0], secp_corpus.OUT_WORDS), np.uint64)
        rc = devcheck.secp_check_run(code, inp.ctypes.data, out.ctypes.data, inp.shape[0])
        assert rc == 0, f"CUDA error {rc}"
        return out
    assert secp_corpus.check(run, op) == len(secp_corpus.cases(op))
