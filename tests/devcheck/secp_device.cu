// Test-only: the arithmetic of phant_b200/csrc/secp256k1.cuh as the GPU runs it -- its PTX carry chains, the asm of mul_wide
// and fp_reduce, __umul64hi -- one case per thread, so that tests/test_gpu_secp_device.py can compare every operation with
// Python integers.  Built by `make -C phant_b200/csrc devcheck` with the library's own flags into
// tests/devcheck/build/libsecp_devcheck.so; nothing in the product links or loads it.
#include <cuda_runtime.h>

#include "../../phant_b200/csrc/secp256k1.cuh"
#include "secp_ops.cuh"

namespace {

__global__ void __launch_bounds__(128) secp_check_kernel(int op, const uint64_t* __restrict__ in, uint64_t* __restrict__ out, uint64_t n)
{
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) secpcheck::run_op(op, in + secpcheck::IN_WORDS * i, out + secpcheck::OUT_WORDS * i);
}

} // namespace

extern "C" void secp_check_layout(int* in_words, int* out_words, int* n_ops)
{
    *in_words = secpcheck::IN_WORDS;
    *out_words = secpcheck::OUT_WORDS;
    *n_ops = secpcheck::N_OPS;
}

// in: n * IN_WORDS words, out: n * OUT_WORDS words (host memory).  The device output starts as 0xA5 bytes, so a word an
// operation fails to write comes back as 0xA5A5A5A5A5A5A5A5.  Returns 0 or the CUDA error code.
extern "C" int secp_check_run(int op, const uint64_t* in, uint64_t* out, uint64_t n)
{
    if (op < 0 || op >= secpcheck::N_OPS) return (int)cudaErrorInvalidValue;
    if (n == 0) return 0;
    const size_t in_bytes = sizeof(uint64_t) * secpcheck::IN_WORDS * n, out_bytes = sizeof(uint64_t) * secpcheck::OUT_WORDS * n;
    uint64_t *d_in = nullptr, *d_out = nullptr;
    cudaError_t e = cudaMalloc(&d_in, in_bytes);
    if (e == cudaSuccess) e = cudaMalloc(&d_out, out_bytes);
    if (e == cudaSuccess) e = cudaMemcpy(d_in, in, in_bytes, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemset(d_out, 0xA5, out_bytes);
    if (e == cudaSuccess) {
        secp_check_kernel<<<(unsigned)((n + 127) / 128), 128>>>(op, d_in, d_out, n);
        e = cudaGetLastError();
    }
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(out, d_out, out_bytes, cudaMemcpyDeviceToHost);
    cudaFree(d_in);
    cudaFree(d_out);
    return (int)e;
}
