// kzg_cells.cu -- EIP-7594 (PeerDAS) cells on the device: the cell extension of a blob (c-kzg compute_cells) and the
// scalars of the batched cell-proof check (verify_cell_kzg_proof_batch, whose pairing lives in bls_pairing.cu):
//   crates/common/crypto/kzg.rs:72-113          verify_cell_kzg_proof_batch, compute_cells
//   crates/common/types/blobs_bundle.rs:152-173 BlobsBundle::verify_kzg_proofs, wrapper version 1
// A blob lists p's values on the 4096 roots of unity in bit-reversed order.  Its extension lists p on the 8192nd roots in
// bit-reversed order: brp13(i) = 2 brp12(i) for i < 4096, so the first half is the blob itself, and brp13(4096 + j) =
// 2 brp12(j) + 1, so the second half is p on the coset w_8192 <w_4096>, again in bit-reversed order.  That half is one
// size-4096 NTT of the coefficients c_i w_8192^i: the zero-padded size-8192 NTT of the spec splits into that and the blob.
// So each blob takes an inverse and a forward NTT of size 4096 (128 KiB of Fr381, one CTA's shared memory), and the
// 256 KiB of the full extension never has to sit in one CTA.
#include "bls12.cuh"
#include <cstring>

namespace b200zk {
namespace {

constexpr uint32_t kN = 4096;       // FIELD_ELEMENTS_PER_BLOB
constexpr uint32_t kExtN = 8192;    // FIELD_ELEMENTS_PER_EXT_BLOB
constexpr uint32_t kCellN = 64;     // FIELD_ELEMENTS_PER_CELL
constexpr uint32_t kCells = 128;    // CELLS_PER_EXT_BLOB
constexpr uint32_t kThreads = 256;  // one CTA per blob: 8 butterflies per thread and stage
constexpr size_t kSmem = kN * 32;   // the blob's 4096 elements

B2_D Fr381 tw_at(const void* tw, uint32_t i) { return load_fe_nc<Fr381>(tw, i); }
B2_D uint32_t brp7(uint32_t c) { return __brev(c) >> 25; }

// tw[i] = w^i for i < 8192, w = 7^((r-1)/8192); tw[8192] = 1/4096 = r - (r-1)/4096.  Montgomery form.  One thread per
// entry, each deriving w from its definition: a one-off per context.  w^2 is the blob domain's root (kzg_roots_build).
__global__ void __launch_bounds__(256) kzg_cells_tw_build(void* __restrict__ tw) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > kExtN) return;
  const uint32_t sh = i == kExtN ? 12 : 13;  // (r - 1) >> sh (r - 1 = r with limb 0 cleared)
  Fr381 e;
#pragma unroll
  for (int k = 0; k < 8; ++k) e.v[k] = ((k ? bls_r_limb(k) : 0u) >> sh) | (k < 7 ? bls_r_limb(k + 1) << (32 - sh) : 0u);
  if (i == kExtN) { store_fe(tw, i, Fr381::to_mont(Fr381::sub(Fr381::zero(), e))); return; }
  Fr381 c = Fr381::zero();
  c.v[0] = 7;
  Fr381 base = Fr381::pow(Fr381::to_mont(c), e.v), acc = Fr381::one();
#pragma unroll 1
  for (uint32_t x = i; x; x >>= 1) {
    if (x & 1) acc = Fr381::mul(acc, base);
    base = Fr381::sqr(base);
  }
  store_fe(tw, i, acc);
}

// In place over the 4096 elements in s, all threads of the CTA, s written and synchronised by the caller.  Twiddles of a
// butterfly span 2h are powers of w_2h = w_8192^(8192 / 2h).  Elements may be canonical or Montgomery: the twiddles are
// Montgomery, so mul keeps the input's form.
// Inverse, Cooley-Tukey: bit-reversed values in, natural-order coefficients out, times 4096 (no scaling)
B2_D void ntt_inverse_brp(uint4* s, const void* tw) {
  for (uint32_t h = 1; h < kN; h <<= 1) {
    const uint32_t step = kExtN / (2 * h);
#pragma unroll 1
    for (uint32_t b = threadIdx.x; b < kN / 2; b += kThreads) {
      const uint32_t j = b & (h - 1), i0 = 2 * b - j, i1 = i0 + h;
      const Fr381 u = load_fe<Fr381>(s, i0), v = Fr381::mul(load_fe<Fr381>(s, i1), tw_at(tw, (kExtN - j * step) & (kExtN - 1)));
      store_fe(s, i0, Fr381::add(u, v));
      store_fe(s, i1, Fr381::sub(u, v));
    }
    __syncthreads();
  }
}
// Forward, Gentleman-Sande: natural-order coefficients in, values on the 4096 roots out in bit-reversed order
B2_D void ntt_forward_brp(uint4* s, const void* tw) {
  for (uint32_t h = kN / 2; h >= 1; h >>= 1) {
    const uint32_t step = kExtN / (2 * h);
#pragma unroll 1
    for (uint32_t b = threadIdx.x; b < kN / 2; b += kThreads) {
      const uint32_t j = b & (h - 1), i0 = 2 * b - j, i1 = i0 + h;
      const Fr381 u = load_fe<Fr381>(s, i0), v = load_fe<Fr381>(s, i1);
      store_fe(s, i0, Fr381::add(u, v));
      store_fe(s, i1, Fr381::mul(Fr381::sub(u, v), tw_at(tw, j * step)));
    }
    __syncthreads();
  }
}

// blob (4096 x 32-byte big-endian, checked < r) -> s as canonical limbs
B2_D void load_blob(uint4* s, const uint8_t* blob) {
  for (uint32_t i = threadIdx.x; i < kN; i += kThreads) store_fe(s, i, load_be32(blob + 32 * i));
  __syncthreads();
}

// One CTA per blob: its 128 cells (8192 x 32-byte big-endian).  Cells 0..63 are the blob's bytes; cells 64..127 are
// the forward NTT of c_i w_8192^i / 4096.  Values stay canonical throughout.
__global__ void __launch_bounds__(kThreads, 1) kzg_cells_extend(const uint8_t* __restrict__ blobs, const void* __restrict__ tw, uint8_t* __restrict__ cells) {
  extern __shared__ uint4 cells_smem[];
  const uint8_t* blob = blobs + (size_t)blockIdx.x * kN * 32;
  uint8_t* out = cells + (size_t)blockIdx.x * kExtN * 32;
  for (uint32_t i = threadIdx.x; i < 2 * kN; i += kThreads)
    reinterpret_cast<uint4*>(out)[i] = __ldg(reinterpret_cast<const uint4*>(blob) + i);
  load_blob(cells_smem, blob);
  ntt_inverse_brp(cells_smem, tw);
  const Fr381 ninv = tw_at(tw, kExtN);
  for (uint32_t i = threadIdx.x; i < kN; i += kThreads)
    store_fe(cells_smem, i, Fr381::mul(Fr381::mul(load_fe<Fr381>(cells_smem, i), tw_at(tw, i)), ninv));
  __syncthreads();
  ntt_forward_brp(cells_smem, tw);
  for (uint32_t i = threadIdx.x; i < kN; i += kThreads) store_be32(out + 32 * (kN + i), load_fe<Fr381>(cells_smem, i));
}

// ---- the batched cell-proof check --------------------------------------------------------------------------------------
// Cell k (global index 128 b + c over blob b, cell c) covers the coset h_c <w_64>, h_c = w_8192^brp7(c), the roots of
// X^64 - s_c with s_c = h_c^64 = w_8192^(64 brp7(c)).  Its interpolation polynomial is I_k = p_b mod (X^64 - s_c):
// coefficient j is sum_m c_b[64 m + j] s_c^m.  With the challenge r,
//   A = sum_k r^k I_k,  A_j = sum_b r^(128 b) sum_m c_b[64 m + j] V_m,  V_m = sum_c r^c s_c^m,
// so one 64 x 64 product per blob gives its share of A, and A of degree < 64 evaluated on the 4096 bit-reversed roots
// is the scalar vector of [A(tau)]1 over the Lagrange setup.

// weights = V_0 .. V_63 (V_0 = sum_c r^c), then r; Montgomery.  One CTA of 65 threads.
__global__ void __launch_bounds__(96) kzg_cells_weights(const uint8_t* __restrict__ r_be, const void* __restrict__ tw, void* __restrict__ weights) {
  const uint32_t m = threadIdx.x;
  if (m > kCellN) return;
  const Fr381 r = Fr381::to_mont(load_be32(r_be));
  if (m == kCellN) { store_fe(weights, m, r); return; }
  Fr381 acc = Fr381::zero(), rc = Fr381::one();
#pragma unroll 1
  for (uint32_t c = 0; c < kCells; ++c) {
    acc = Fr381::add(acc, Fr381::mul(rc, tw_at(tw, (kCellN * brp7(c) * m) & (kExtN - 1))));
    rc = Fr381::mul(rc, r);
  }
  store_fe(weights, m, acc);
}

// One CTA per blob: partial[64 b + j] = r^(128 b) / 4096 sum_m c'_b[64 m + j] V_m (canonical), c' = 4096 c the unscaled
// inverse NTT
__global__ void __launch_bounds__(kThreads, 1) kzg_cells_interp(const uint8_t* __restrict__ blobs, const void* __restrict__ tw, const void* __restrict__ weights,
                                                               void* __restrict__ partial) {
  extern __shared__ uint4 cells_smem[];
  __shared__ uint4 s_scale[2];
  if (threadIdx.x == 0) {
    const uint32_t e[8] = {kCells * blockIdx.x, 0, 0, 0, 0, 0, 0, 0};
    store_fe(s_scale, 0, Fr381::mul(Fr381::pow(load_fe_nc<Fr381>(weights, kCellN), e), tw_at(tw, kExtN)));
  }
  load_blob(cells_smem, blobs + (size_t)blockIdx.x * kN * 32);
  ntt_inverse_brp(cells_smem, tw);
  const uint32_t j = threadIdx.x;
  if (j >= kCellN) return;
  Fr381 acc = Fr381::zero();
#pragma unroll 1
  for (uint32_t m = 0; m < kN / kCellN; ++m) acc = Fr381::add(acc, Fr381::mul(load_fe<Fr381>(cells_smem, kCellN * m + j), load_fe_nc<Fr381>(weights, m)));
  store_fe(partial, (size_t)kCellN * blockIdx.x + j, Fr381::mul(acc, load_fe<Fr381>(s_scale, 0)));
}

// One CTA: A_j = sum_b partial[64 b + j], zero-padded to 4096 and evaluated on the bit-reversed roots; out: canonical
// little-endian limbs, the scalars of the Lagrange-setup MSM
__global__ void __launch_bounds__(kThreads, 1) kzg_cells_interp_eval(const void* __restrict__ partial, size_t n, const void* __restrict__ tw, void* __restrict__ s_setup) {
  extern __shared__ uint4 cells_smem[];
  for (uint32_t i = threadIdx.x; i < kN; i += kThreads) {
    Fr381 a = Fr381::zero();
    if (i < kCellN)
      for (size_t b = 0; b < n; ++b) a = Fr381::add(a, load_fe<Fr381>(partial, kCellN * b + i));
    store_fe(cells_smem, i, a);
  }
  __syncthreads();
  ntt_forward_brp(cells_smem, tw);
  for (uint32_t i = threadIdx.x; i < kN; i += kThreads) store_fe(s_setup, i, load_fe<Fr381>(cells_smem, i));
}

// k < n: s_lin[k] = r^(128 k) V_0, commitment k's scalar; n <= k < 129 n, cell q = k - n: s_lin[k] = r^q s_(q mod 128)
// and s_proof[q] = r^q.  Canonical little-endian limbs.
__global__ void __launch_bounds__(256) kzg_cells_scalars(const void* __restrict__ tw, const void* __restrict__ weights, size_t n,
                                                         void* __restrict__ s_proof, void* __restrict__ s_lin) {
  const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (k >= (kCells + 1) * n) return;
  const size_t q = k < n ? kCells * k : k - n;
  const uint32_t e[8] = {(uint32_t)q, (uint32_t)((uint64_t)q >> 32), 0, 0, 0, 0, 0, 0};
  const Fr381 rq = Fr381::pow(load_fe_nc<Fr381>(weights, kCellN), e);
  if (k < n) { store_fe(s_lin, k, Fr381::from_mont(Fr381::mul(rq, load_fe_nc<Fr381>(weights, 0)))); return; }
  store_fe(s_proof, q, Fr381::from_mont(rq));
  store_fe(s_lin, k, Fr381::from_mont(Fr381::mul(rq, tw_at(tw, kCellN * brp7((uint32_t)(q % kCells))))));
}

// the twiddle table, built on first use; later calls on any stream wait on its event
int cells_tw(b200zk_ctx* ctx, cudaStream_t st, const void** tw) {
  if (!ctx->kzg_cells_tw.p) {
    B2_TRY(ensure(ctx, ctx->kzg_cells_tw, (kExtN + 1) * 32));
    B2_LAUNCH(ctx, kzg_cells_tw_build, (kExtN + 256) / 256, 256, 0, st, ctx->kzg_cells_tw.p);
    if (cudaEventCreateWithFlags(&ctx->kzg_cells_tw_ready, cudaEventDisableTiming) == cudaSuccess) B2_CUDA(ctx, cudaEventRecord(ctx->kzg_cells_tw_ready, st));
    else { cudaGetLastError(); ctx->kzg_cells_tw_ready = nullptr; B2_CUDA(ctx, cudaStreamSynchronize(st)); }
  } else if (ctx->kzg_cells_tw_ready) {
    B2_CUDA(ctx, cudaStreamWaitEvent(st, ctx->kzg_cells_tw_ready, 0));
  }
  if (!ctx->attr_kzg_cells) {
    B2_CUDA(ctx, cudaFuncSetAttribute(kzg_cells_extend, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
    B2_CUDA(ctx, cudaFuncSetAttribute(kzg_cells_interp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
    B2_CUDA(ctx, cudaFuncSetAttribute(kzg_cells_interp_eval, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
    ctx->attr_kzg_cells = true;
  }
  *tw = ctx->kzg_cells_tw.p;
  return B200ZK_OK;
}

}  // namespace

int kzg_cells_run(b200zk_ctx* ctx, const uint8_t* d_blobs, size_t n, uint8_t* d_cells, cudaStream_t st) {
  const void* tw = nullptr;
  B2_TRY(cells_tw(ctx, st, &tw));
  B2_LAUNCH(ctx, kzg_cells_extend, (unsigned)n, kThreads, kSmem, st, d_blobs, tw, d_cells);
  return B200ZK_OK;
}

int kzg_cell_scalars_run(b200zk_ctx* ctx, const uint8_t* d_blobs, size_t n, const uint8_t* d_r_be, void* d_weights, void* d_partial,
                         void* d_s_proof, void* d_s_lin, void* d_s_setup, cudaStream_t st) {
  const void* tw = nullptr;
  B2_TRY(cells_tw(ctx, st, &tw));
  B2_LAUNCH(ctx, kzg_cells_weights, 1, 96, 0, st, d_r_be, tw, d_weights);
  B2_LAUNCH(ctx, kzg_cells_interp, (unsigned)n, kThreads, kSmem, st, d_blobs, tw, (const void*)d_weights, d_partial);
  B2_LAUNCH(ctx, kzg_cells_interp_eval, 1, kThreads, kSmem, st, (const void*)d_partial, n, tw, d_s_setup);
  B2_LAUNCH(ctx, kzg_cells_scalars, (unsigned)(((kCells + 1) * n + 255) / 256), 256, 0, st, tw, (const void*)d_weights, n, d_s_proof, d_s_lin);
  return B200ZK_OK;
}

}  // namespace b200zk

using namespace b200zk;

extern "C" {

int b200zk_kzg_compute_cells(b200zk_ctx* ctx, const uint8_t* blobs, size_t n_blobs, uint8_t* cells) {
  static const char* what = "kzg_compute_cells";
  if (!ctx || (n_blobs && (!blobs || !cells))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_compute_cells: null argument");
  NvtxRange nvtx("b200zk:kzg_compute_cells");
  DeviceGuard guard(ctx);
  if (!n_blobs) return B200ZK_OK;
  cudaStream_t st = ctx->stream;
  uint8_t *d_blobs, *d_cells;
  Carve c;
  for (int pass = 0; pass < 2; ++pass) {
    if (pass) { B2_TRY(ensure(ctx, ctx->ws_kzg, c.off + 256)); c = Carve{(uint8_t*)ctx->ws_kzg.p, 0}; }
    d_blobs = c.take<uint8_t>(n_blobs * kN * 32); d_cells = c.take<uint8_t>(n_blobs * kExtN * 32);
  }
  B2_CUDA(ctx, cudaMemcpyAsync(d_blobs, blobs, n_blobs * kN * 32, cudaMemcpyHostToDevice, st));
  size_t bad = 0;
  B2_TRY(bls_scalars_check(ctx, d_blobs, n_blobs * kN, true, st, &bad));
  if (bad < n_blobs * kN) {
    char msg[160];
    snprintf(msg, sizeof msg, "%s: blob %zu, element %zu is >= the BLS12-381 group order", what, bad / kN, bad % kN);
    return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, msg);
  }
  B2_TRY(kzg_cells_run(ctx, d_blobs, n_blobs, d_cells, st));
  B2_CUDA(ctx, cudaMemcpyAsync(cells, d_cells, n_blobs * kExtN * 32, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

}  // extern "C"
