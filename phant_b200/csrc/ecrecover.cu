// ecrecover.cu -- batched transaction-sender recovery (row N4 of SURVEY.md 8f): for every (message hash, signature)
// the secp256k1 public key and the address keccak256(pubkey[1..])[12..], one signature per thread.
//
// Replaces, for a whole block at once, the per-transaction tail of TxSigner.get_sender (reference
// src/signer/signer.zig:78-79: ecdsa_signer.erecover + hasher.keccak256).  The curve arithmetic is secp256k1.cuh, the hash
// is the same sponge the batched Keccak kernel uses (keccak_f1600.cuh) -- recovery and hashing are fused: the public key
// never leaves the thread before it has been turned into the address.
#include "../../include/phant_gpu.h"
#include "common.cuh"
#include "ctx.cuh"
#include "keccak_f1600.cuh"
#include "secp256k1.cuh"

using namespace phant;

#define CU(expr)                                                              \
    do {                                                                      \
        cudaError_t e_ = (expr);                                              \
        if (e_ != cudaSuccess) return ctx->fail(e_, #expr, __FILE__, __LINE__); \
    } while (0)

namespace {

__global__ void __launch_bounds__(128)
ecrecover_kernel(const uint8_t* __restrict__ hashes32, const uint8_t* __restrict__ sigs65, uint64_t n, uint8_t* __restrict__ pubkeys65,
                 uint8_t* __restrict__ addresses20, uint8_t* __restrict__ ok)
{
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint8_t h[32], sig[65];
        __align__(8) uint8_t pub[64];
        for (int b = 0; b < 32; ++b) h[b] = hashes32[32 * i + b];
        for (int b = 0; b < 65; ++b) sig[b] = sigs65[65 * i + b];
        const bool good = secp::ecrecover(h, sig, pub);
        if (!good)
            for (int b = 0; b < 64; ++b) pub[b] = 0;
        if (pubkeys65) {
            pubkeys65[65 * i] = good ? 0x04 : 0x00;
            for (int b = 0; b < 64; ++b) pubkeys65[65 * i + 1 + b] = pub[b];
        }
        if (addresses20) {
            uint64_t dg[4] = {0, 0, 0, 0};
            if (good) keccak256_thread<2>(pub, 64, dg);
            for (int b = 0; b < 20; ++b) addresses20[20 * i + b] = good ? (uint8_t)(dg[(12 + b) >> 3] >> (8 * ((12 + b) & 7))) : 0;
        }
        ok[i] = good ? 1 : 0;
    }
}

} // namespace

extern "C" int phant_gpu_ecrecover_batch(phant_gpu_ctx* ctx, const uint8_t* hashes32, const uint8_t* sigs65, uint64_t n,
                                         uint8_t* pubkeys65, uint8_t* addresses20, uint8_t* ok)
{
    if (!ctx || (n && (!hashes32 || !sigs65 || !ok))) return PHANT_GPU_E_INVALID;
    if (n == 0) return PHANT_GPU_OK;
    CU(cudaSetDevice(ctx->device));
    cudaStream_t s = ctx->stream;
    const bool dev = ctx->flags & PHANT_GPU_FLAG_DEVICE_PTRS;
    const uint8_t* d_h = hashes32; const uint8_t* d_s = sigs65;
    uint8_t* d_pub = pubkeys65; uint8_t* d_addr = addresses20; uint8_t* d_ok = ok;
    if (!dev) {
        uint8_t *h, *sig;
        if (int rc = carve(ctx, ctx->d_msgs, [&](Carve& c) {
                h = c.take<uint8_t>(32 * n); sig = c.take<uint8_t>(65 * n);
                d_pub = pubkeys65 ? c.take<uint8_t>(65 * n) : nullptr; d_addr = addresses20 ? c.take<uint8_t>(20 * n) : nullptr;
                d_ok = c.take<uint8_t>(n);
            })) return rc;
        CU(cudaMemcpyAsync(h, hashes32, 32 * n, cudaMemcpyHostToDevice, s));
        CU(cudaMemcpyAsync(sig, sigs65, 65 * n, cudaMemcpyHostToDevice, s));
        ctx->stats.h2d_bytes += 97 * n;
        d_h = h; d_s = sig;
    }
    uint64_t blocks = (n + 127) / 128;
    const uint64_t cap = (uint64_t)keccak_num_sms(ctx->device) * 8;
    if (blocks > cap) blocks = cap;
    ecrecover_kernel<<<(unsigned)blocks, 128, 0, s>>>(d_h, d_s, n, d_pub, d_addr, d_ok);
    CU(cudaGetLastError());
    ctx->stats.launches++;
    if (dev) return PHANT_GPU_OK;
    if (int rc = copy_out(ctx, pubkeys65, d_pub, 65 * n)) return rc;
    if (int rc = copy_out(ctx, addresses20, d_addr, 20 * n)) return rc;
    if (int rc = copy_out(ctx, ok, d_ok, n)) return rc;
    CU(cudaStreamSynchronize(s));
    return PHANT_GPU_OK;
}
