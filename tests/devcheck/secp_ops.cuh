// Test-only: one case of one operation of phant_b200/csrc/secp256k1.cuh, for the device build (tests/devcheck/secp_device.cu)
// and the host build (tests/hostcheck/ecrecover_host.cpp) alike, so that both branches of the header's `#if
// defined(__CUDA_ARCH__)` are held to the same cases by tests/secp_corpus.py.  Include after secp256k1.cuh.
//
// A case is IN_WORDS little-endian 64-bit words in and OUT_WORDS out; 256-bit values are four words, low limb first.
//   ADD_RAW, SUB_RAW   in a, b          out r, carry or borrow word (out[4])
//   MUL_WIDE           in a, b          out the 8 limbs of a * b
//   FP_REDUCE          in t (8 limbs)   out t mod p
//   FP_ADD .. SC_INV   in a (, b)       out the result
//   JAC_DOUBLE         in X, Y, Z       out X, Y, Z
//   JAC_ADD_AFFINE     in X, Y, Z, qx, qy  out X, Y, Z
//   TO_AFFINE          in X, Y, Z       out x, y, inf (out[8])
//   ECRECOVER          in z (the hash as an integer), r, s, recid (in[12])  out X, Y, ok (out[8])
#pragma once
#include <stdint.h>

namespace secpcheck {

enum Op {
    ADD_RAW = 0, SUB_RAW, MUL_WIDE, FP_REDUCE, FP_ADD, FP_SUB, FP_NEG, FP_MUL, FP_INV, FP_SQRT_CANDIDATE, SC_MUL, SC_NEG, SC_INV,
    JAC_DOUBLE, JAC_ADD_AFFINE, TO_AFFINE, ECRECOVER, N_OPS
};
constexpr int IN_WORDS = 20, OUT_WORDS = 13;

using namespace phant::secp;

__device__ __forceinline__ u256 ld(const uint64_t* w) { return u256{{w[0], w[1], w[2], w[3]}}; }
__device__ __forceinline__ void st(uint64_t* w, const u256& a)
{
    for (int i = 0; i < 4; ++i) w[i] = a.v[i];
}
__device__ __forceinline__ void st_jac(uint64_t* w, const Jac& p)
{
    st(w, p.x); st(w + 4, p.y); st(w + 8, p.z);
}

__device__ __noinline__ void run_op(int op, const uint64_t* in, uint64_t* out)
{
    const u256 a = ld(in), b = ld(in + 4);
    const Jac jp{ld(in), ld(in + 4), ld(in + 8)};
    switch (op) {
    case ADD_RAW: { u256 r; out[4] = add_raw(r, a, b); st(out, r); break; }
    case SUB_RAW: { u256 r; out[4] = sub_raw(r, a, b); st(out, r); break; }
    case MUL_WIDE: {
        uint64_t t[8];
        mul_wide(t, a, b);
        for (int i = 0; i < 8; ++i) out[i] = t[i];
        break;
    }
    case FP_REDUCE: {
        uint64_t t[8];
        for (int i = 0; i < 8; ++i) t[i] = in[i];
        st(out, fp_reduce(t));
        break;
    }
    case FP_ADD: st(out, fp_add(a, b)); break;
    case FP_SUB: st(out, fp_sub(a, b)); break;
    case FP_NEG: st(out, fp_neg(a)); break;
    case FP_MUL: st(out, fp_mul(a, b)); break;
    case FP_INV: st(out, fp_inv(a)); break;
    case FP_SQRT_CANDIDATE: st(out, fp_sqrt_candidate(a)); break;
    case SC_MUL: st(out, sc_mul(a, b)); break;
    case SC_NEG: st(out, sc_neg(a)); break;
    case SC_INV: st(out, sc_inv(a)); break;
    case JAC_DOUBLE: st_jac(out, jac_double(jp)); break;
    case JAC_ADD_AFFINE: st_jac(out, jac_add_affine(jp, Affine{ld(in + 12), ld(in + 16), false})); break;
    case TO_AFFINE: {
        const Affine q = to_affine(jp);
        st(out, q.x); st(out + 4, q.y);
        out[8] = q.inf ? 1 : 0;
        break;
    }
    case ECRECOVER: {
        uint8_t h[32], sig[65], pub[64];
        to_be(h, ld(in));
        to_be(sig, ld(in + 4));
        to_be(sig + 32, ld(in + 8));
        sig[64] = (uint8_t)in[12];
        const bool ok = ecrecover(h, sig, pub);
        st(out, ok ? from_be(pub) : u256{{0, 0, 0, 0}});
        st(out + 4, ok ? from_be(pub + 32) : u256{{0, 0, 0, 0}});
        out[8] = ok ? 1 : 0;
        break;
    }
    default: break;
    }
}

} // namespace secpcheck
