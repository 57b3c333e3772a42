// secp256k1.cu -- batched ECRECOVER on the device: Crypto::secp256k1_ecrecover and Crypto::recover_signer of the
// reference (crates/common/crypto/provider.rs:63-171), `count` independent items per call, one thread per item.
// The arithmetic, the curve, Keccak and the rules of each check are in secp256k1.cuh; this file holds the kernels, the
// per-context table of G multiples and the C entry point.
#include "common.cuh"
#include "secp256k1.cuh"

namespace b200zk {
namespace {

static_assert(kSecpLowS == B200ZK_ECRECOVER_LOW_S, "secp256k1.cuh and b200zk.h disagree on the low-s flag");
constexpr int kRecoverThreads = 128;

// table[d - 1] = d G for d = 1 .. 255, one thread per entry; built once per context
__global__ void __launch_bounds__(256) secp256k1_gtab_build(Affine<SecpFp>* table) {
  const uint32_t d = blockIdx.x * blockDim.x + threadIdx.x + 1;
  if (d > kSecpGTable) return;
  table[d - 1] = secp_g_multiple(d);
}

// one thread per item: sigs 65 B, msgs 32 B, out 32 B, status 1 B each
__global__ void __launch_bounds__(kRecoverThreads) secp256k1_ecrecover_kernel(const uint8_t* __restrict__ sigs, const uint8_t* __restrict__ msgs, size_t n,
                                                                              uint32_t flags, const Affine<SecpFp>* __restrict__ gtab,
                                                                              uint8_t* __restrict__ out, uint8_t* __restrict__ status) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  alignas(16) uint8_t h[32];
  status[i] = (uint8_t)secp_recover(sigs + 65 * i, msgs + 32 * i, flags, gtab, h);
  uint4* dst = reinterpret_cast<uint4*>(out + 32 * i);  // out is 256-byte aligned (Carve), items 32 B apart
  const uint32_t* w = reinterpret_cast<const uint32_t*>(h);
  dst[0] = make_uint4(w[0], w[1], w[2], w[3]);
  dst[1] = make_uint4(w[4], w[5], w[6], w[7]);
}

// the G table, built on first use
int secp_gtab(b200zk_ctx* ctx, cudaStream_t st, const void** table) {
  return once_table(ctx, ctx->secp_gtab, kSecpGTable * sizeof(Affine<SecpFp>), st, [&](void* t) -> int {
    B2_LAUNCH(ctx, secp256k1_gtab_build, (kSecpGTable + 255) / 256, 256, 0, st, (Affine<SecpFp>*)t);
    return B200ZK_OK;
  }, table);
}

}  // namespace
}  // namespace b200zk

using namespace b200zk;

extern "C" {

int b200zk_secp256k1_ecrecover_batch(b200zk_ctx* ctx, const uint8_t* sigs, const uint8_t* msgs, size_t count, uint32_t flags, uint8_t* out,
                                     uint8_t* status) {
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  if (flags & ~(uint32_t)B200ZK_ECRECOVER_LOW_S) return fail(ctx, B200ZK_ERR_INVALID_ARG, "secp256k1_ecrecover_batch: unknown flag bits");
  if (count && (!sigs || !msgs || !out || !status)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "secp256k1_ecrecover_batch: null argument");
  NvtxRange nvtx("b200zk:secp256k1_ecrecover_batch");
  DeviceGuard guard(ctx);
  if (!count) return B200ZK_OK;
  cudaStream_t st = ctx->stream;
  const void* gtab;
  B2_TRY(secp_gtab(ctx, st, &gtab));
  uint8_t *dsig, *dmsg, *dout, *dst;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    dsig = c.take<uint8_t>(65 * count); dmsg = c.take<uint8_t>(32 * count); dout = c.take<uint8_t>(32 * count); dst = c.take<uint8_t>(count);
  }));
  B2_CUDA(ctx, cudaMemcpyAsync(dsig, sigs, 65 * count, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(dmsg, msgs, 32 * count, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, secp256k1_ecrecover_kernel, (unsigned)((count + kRecoverThreads - 1) / kRecoverThreads), kRecoverThreads, 0, st,
            (const uint8_t*)dsig, (const uint8_t*)dmsg, count, flags, (const Affine<SecpFp>*)gtab, dout, dst);
  B2_CUDA(ctx, cudaMemcpyAsync(out, dout, 32 * count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(status, dst, count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

}  // extern "C"
