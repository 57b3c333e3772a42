// secp256r1.cu -- batched P256VERIFY on the device: Crypto::secp256r1_verify of the reference
// (crates/common/crypto/provider.rs:415-459, levm p_256_verify, EIP-7951), `count` independent items per call, one thread
// per item.  The arithmetic, the curve and the rules of each check are in secp256r1.cuh; this file holds the kernels, the
// per-context table of G multiples and the C entry point.
#include "common.cuh"
#include "secp256r1.cuh"

namespace b200zk {
namespace {

constexpr int kVerifyThreads = 128;

// table[d - 1] = d G for d = 1 .. 4095, one thread per entry; built once per context
__global__ void __launch_bounds__(256) secp256r1_gtab_build(Affine<P256Fp>* table) {
  const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x + 1;
  if (d > kSecpGTable) return;
  table[d - 1] = p256_g_multiple(d);
}

// one thread per item: 160 input bytes, one result byte (1 = verified)
__global__ void __launch_bounds__(kVerifyThreads) secp256r1_verify_kernel(const uint8_t* __restrict__ inputs, size_t n,
                                                                           const Affine<P256Fp>* __restrict__ gtab, uint8_t* __restrict__ result) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  result[i] = p256_verify(inputs + 160 * i, gtab) ? 1 : 0;
}

// the G table, built on first use
int p256_gtab(b200zk_ctx* ctx, cudaStream_t st, const void** table) {
  return once_table(ctx, ctx->p256_gtab, kSecpGTable * sizeof(Affine<P256Fp>), st, [&](void* t) -> int {
    B2_LAUNCH(ctx, secp256r1_gtab_build, (kSecpGTable + 255) / 256, 256, 0, st, (Affine<P256Fp>*)t);
    return B200ZK_OK;
  }, table);
}

}  // namespace
}  // namespace b200zk

using namespace b200zk;

extern "C" {

int b200zk_secp256r1_verify_batch(b200zk_ctx* ctx, const uint8_t* inputs, size_t count, uint8_t* result) {
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  if (count && (!inputs || !result)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "secp256r1_verify_batch: null argument");
  NvtxRange nvtx("b200zk:secp256r1_verify_batch");
  DeviceGuard guard(ctx);
  if (!count) return B200ZK_OK;
  cudaStream_t st = ctx->stream;
  const void* gtab;
  B2_TRY(p256_gtab(ctx, st, &gtab));
  uint8_t *din, *dres;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) { din = c.take<uint8_t>(160 * count); dres = c.take<uint8_t>(count); }));
  B2_CUDA(ctx, cudaMemcpyAsync(din, inputs, 160 * count, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, secp256r1_verify_kernel, (unsigned)((count + kVerifyThreads - 1) / kVerifyThreads), kVerifyThreads, 0, st,
            (const uint8_t*)din, count, (const Affine<P256Fp>*)gtab, dres);
  B2_CUDA(ctx, cudaMemcpyAsync(result, dres, count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

}  // extern "C"
