// Test-only: phant_b200/csrc/secp256k1.cuh (the per-thread device function of the ecrecover kernel) compiled as HOST code
// so that its arithmetic can be checked against the oracle and OpenSSL on a machine without a GPU.  Built as a shared
// object by tests/test_ecrecover_header_host.py; nothing in the product links or loads this.
#include <stdint.h>
#define __device__
#define __forceinline__ inline
#define __noinline__
#include "../../phant_b200/csrc/secp256k1.cuh"
#include "../devcheck/secp_ops.cuh"

extern "C" int host_ecrecover(const uint8_t* hash32, const uint8_t* sig65, uint8_t* pub65)
{
    pub65[0] = 0x04;
    return phant::secp::ecrecover(hash32, sig65, pub65 + 1) ? 1 : 0;
}
extern "C" void host_fp_mul(const uint8_t* a32, const uint8_t* b32, uint8_t* out32)
{
    using namespace phant::secp;
    to_be(out32, fp_mul(from_be(a32), from_be(b32)));
}
extern "C" void host_sc_mul(const uint8_t* a32, const uint8_t* b32, uint8_t* out32)
{
    using namespace phant::secp;
    to_be(out32, sc_mul(from_be(a32), from_be(b32)));
}
extern "C" void host_fp_addsub(const uint8_t* a32, const uint8_t* b32, uint8_t* sum32, uint8_t* diff32)
{
    using namespace phant::secp;
    to_be(sum32, fp_add(from_be(a32), from_be(b32)));
    to_be(diff32, fp_sub(from_be(a32), from_be(b32)));
}

// the cases of tests/secp_corpus.py through the `#else` branches (same layout as tests/devcheck/secp_device.cu)
extern "C" void secp_check_layout(int* in_words, int* out_words, int* n_ops)
{
    *in_words = secpcheck::IN_WORDS;
    *out_words = secpcheck::OUT_WORDS;
    *n_ops = secpcheck::N_OPS;
}
extern "C" int secp_check_run(int op, const uint64_t* in, uint64_t* out, uint64_t n)
{
    if (op < 0 || op >= secpcheck::N_OPS) return 1;
    for (uint64_t i = 0; i < n * secpcheck::OUT_WORDS; ++i) out[i] = 0xA5A5A5A5A5A5A5A5ull;
    for (uint64_t i = 0; i < n; ++i) secpcheck::run_op(op, in + secpcheck::IN_WORDS * i, out + secpcheck::OUT_WORDS * i);
    return 0;
}
