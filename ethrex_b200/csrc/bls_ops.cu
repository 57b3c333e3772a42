// bls_ops.cu -- EIP-2537 G1/G2 addition and multi-scalar multiplication on the device, `count` items per call: the Prague
// precompiles 0x0b-0x0e behind the reference's Crypto::{bls12_381_g1_add, _g1_msm, _g2_add, _g2_msm}
// (/root/reference/crates/common/crypto/provider.rs:549-640; levm precompiles.rs:1056-1315).
//
// Every kernel is one template over the coordinate field, Fp381 (G1) or Fp2_381 (G2, the twist): the XYZZ formulas of
// curve.cuh, affine_on_curve and xyzz_scalar_mul instantiate over both.
//   add:        one thread per item: range and padding, on-curve, one mixed XYZZ addition (identity, doubling and P + (-P)
//               handled), normalise, encode.  No subgroup check (EIP-2537 asks none for addition).
//   MSM terms:  one thread per pair: range and padding, on-curve, r P = O, then k P by double-and-add over the raw 256-bit
//               scalar (k P = (k mod r) P in the subgroup, so no reduction).  The subgroup check costs as much as the term,
//               so every point's work is one thread's; Pippenger would share nothing here.
//   MSM fold:   one CTA per call: a strided XYZZ sum per thread, then a tree in shared memory, then one normalisation.
#include "bls12.cuh"

namespace b200zk {
namespace {

typedef Fp2_381 F2;

constexpr int kFoldThreads = 64;  // XYZZ<F2> is 384 B: the fold tree of a G2 call holds 24 KB of shared memory

template <class F> B2_HD constexpr size_t fe_bytes() { return 64 * (sizeof(F) / sizeof(Fp381)); }  // EIP-2537 bytes of one coordinate
template <class F> B2_HD constexpr size_t point_bytes() { return 2 * fe_bytes<F>(); }                // 128 (G1) / 256 (G2)
template <class F> B2_HD constexpr size_t pair_bytes() { return point_bytes<F>() + 32; }              // point | 32-byte big-endian scalar

// EIP-2537 coordinate -> Montgomery form; false on a nonzero padding byte or a value >= p
B2_D bool load_fe64(const uint8_t* src, Fp381* out) {
  Fp381 c;
  const bool ok = load_fp64(src, &c);
  *out = Fp381::to_mont(c);
  return ok;
}
B2_D bool load_fe64(const uint8_t* src, F2* out) { return load_fe64(src, &out->c0) & load_fe64(src + 64, &out->c1); }

// both coordinates are range-checked whatever the first one gave, so status 2 never depends on the order of the checks
template <class F> B2_D bool load_point64(const uint8_t* src, Affine<F>* p) { return load_fe64(src, &p->x) & load_fe64(src + fe_bytes<F>(), &p->y); }

B2_D void store_fe64(uint8_t* out, const Fp381& a) {
  uint32_t* w = reinterpret_cast<uint32_t*>(out);
  w[0] = w[1] = w[2] = w[3] = 0;
  store_be48(out + 16, Fp381::from_mont(a));
}
B2_D void store_fe64(uint8_t* out, const F2& a) { store_fe64(out, a.c0); store_fe64(out + 64, a.c1); }

// the precompile's output: padded EIP-2537 coordinates, the identity (0, 0) as all-zero bytes
template <class F> B2_D void store_point64(uint8_t* out, const Affine<F>& p) { store_fe64(out, p.x); store_fe64(out + fe_bytes<F>(), p.y); }

template <class F> B2_D bool in_subgroup(const Affine<F>& p) {
  if constexpr (sizeof(F) == sizeof(Fp381)) return g1_in_subgroup(p);
  else return g2_in_subgroup(p);
}

// ---- kernels ----------------------------------------------------------------------------------------------------------
// one thread per item: out[i] = a[i] + b[i].  Both points are range-checked (status 2) before either curve check (status 3)
template <class F>
__global__ void __launch_bounds__(64) bls_add(const uint8_t* __restrict__ a, const uint8_t* __restrict__ b, size_t n, uint8_t* out, uint8_t* st) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<F> p, q, r = {F::zero(), F::zero()};
  uint32_t s;
  if (!(load_point64(a + point_bytes<F>() * i, &p) & load_point64(b + point_bytes<F>() * i, &q))) s = B200ZK_ERR_NOT_IN_FIELD;
  else if (!affine_on_curve(p) || !affine_on_curve(q)) s = B200ZK_ERR_NOT_ON_CURVE;
  else {
    XYZZ<F> acc = xyzz_from_affine(p);
    xyzz_add_mixed(acc, q.x, q.y);
    r = xyzz_to_affine(acc);
    s = r.is_inf() ? B200ZK_OK_INFINITY : B200ZK_OK;
  }
  store_point64(out + point_bytes<F>() * i, r);
  st[i] = (uint8_t)s;
}

// one thread per (point, scalar) pair: terms[i] = k P, pst[i] = 0, 2 (range, padding) or 3 (off the curve or outside the
// order-r subgroup; checked for the identity-free points whatever the scalar, as the provider's is_torsion_free)
template <class F>
__global__ void __launch_bounds__(64) bls_msm_terms(const uint8_t* __restrict__ pairs, size_t n, XYZZ<F>* terms, uint8_t* pst) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* src = pairs + pair_bytes<F>() * i;
  Affine<F> p;
  XYZZ<F> t = XYZZ<F>::identity();
  uint32_t s = 0;
  if (!load_point64(src, &p)) s = B200ZK_ERR_NOT_IN_FIELD;
  else if (!affine_on_curve(p) || (!p.is_inf() && !in_subgroup(p))) s = B200ZK_ERR_NOT_ON_CURVE;
  else if (!p.is_inf()) t = xyzz_scalar_mul<F>(load_be32(src + point_bytes<F>()).v, p);  // raw 256 bits, not reduced
  terms[i] = t;
  pst[i] = (uint8_t)s;
}

// one CTA per call: pairs [offsets[c], offsets[c + 1]).  A range error anywhere in the call outranks a curve error (the
// precedence of bls_pairing_final); a failed call writes zero bytes
template <class F>
__global__ void __launch_bounds__(kFoldThreads) bls_msm_fold(const XYZZ<F>* terms, const uint8_t* pst, const uint32_t* offsets, uint8_t* out, uint8_t* status) {
  __shared__ XYZZ<F> part[kFoldThreads];
  const uint32_t c = blockIdx.x, t = threadIdx.x, lo = offsets[c], hi = offsets[c + 1];
  bool range = false, curve = false;
  for (uint32_t k = lo + t; k < hi; k += kFoldThreads) {
    const uint8_t ps = pst[k];
    range |= ps == B200ZK_ERR_NOT_IN_FIELD;
    curve |= ps == B200ZK_ERR_NOT_ON_CURVE;
  }
  range = __syncthreads_or(range);
  curve = __syncthreads_or(curve);
  uint8_t* dst = out + point_bytes<F>() * c;
  if (range || curve) {
    if (t == 0) {
      store_point64(dst, Affine<F>{F::zero(), F::zero()});
      status[c] = range ? B200ZK_ERR_NOT_IN_FIELD : B200ZK_ERR_NOT_ON_CURVE;
    }
    return;
  }
  XYZZ<F> acc = XYZZ<F>::identity();
#pragma unroll 1
  for (uint32_t k = lo + t; k < hi; k += kFoldThreads) xyzz_add(acc, terms[k]);
  part[t] = acc;
  __syncthreads();
#pragma unroll 1
  for (uint32_t h = kFoldThreads / 2; h > 0; h >>= 1) {
    if (t < h) {
      acc = part[t];
      xyzz_add(acc, part[t + h]);
      part[t] = acc;
    }
    __syncthreads();
  }
  if (t == 0) {
    const Affine<F> r = xyzz_to_affine(part[0]);
    store_point64(dst, r);
    status[c] = r.is_inf() ? B200ZK_OK_INFINITY : B200ZK_OK;
  }
}

// ---- host side ----------------------------------------------------------------------------------------------------------
template <class F>
int add_batch(b200zk_ctx* ctx, const char* what, const uint8_t* a, const uint8_t* b, size_t count, uint8_t* out, uint8_t* status) {
  const std::string w = what;
  if (!ctx || (count && (!a || !b || !out || !status))) return fail(ctx, B200ZK_ERR_INVALID_ARG, (w + ": null argument").c_str());
  NvtxRange nvtx(("b200zk:" + w).c_str());
  DeviceGuard guard(ctx);
  if (!count) return B200ZK_OK;
  constexpr size_t kPt = point_bytes<F>();
  cudaStream_t st = ctx->stream;
  uint8_t *da, *db, *dout, *dst;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    da = c.take<uint8_t>(kPt * count); db = c.take<uint8_t>(kPt * count); dout = c.take<uint8_t>(kPt * count); dst = c.take<uint8_t>(count);
  }));
  B2_CUDA(ctx, cudaMemcpyAsync(da, a, kPt * count, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(db, b, kPt * count, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, bls_add<F>, (unsigned)((count + 63) / 64), 64, 0, st, (const uint8_t*)da, (const uint8_t*)db, count, dout, dst);
  B2_CUDA(ctx, cudaMemcpyAsync(out, dout, kPt * count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(status, dst, count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

template <class F>
int msm_batch(b200zk_ctx* ctx, const char* what, const uint8_t* pairs, const uint32_t* pair_offsets, size_t count, uint8_t* out, uint8_t* status) {
  const std::string w = what;
  if (!ctx || (count && (!pair_offsets || !out || !status))) return fail(ctx, B200ZK_ERR_INVALID_ARG, (w + ": null argument").c_str());
  if (count && pair_offsets[count] && !pairs) return fail(ctx, B200ZK_ERR_INVALID_ARG, (w + ": null pairs").c_str());
  NvtxRange nvtx(("b200zk:" + w).c_str());
  DeviceGuard guard(ctx);
  if (!count) return B200ZK_OK;
  B2_TRY(check_offsets(ctx, pair_offsets, count, what));
  const size_t n = pair_offsets[count];
  constexpr size_t kPt = point_bytes<F>(), kPair = pair_bytes<F>();
  cudaStream_t st = ctx->stream;
  uint8_t *in, *pst, *dout, *dst;
  XYZZ<F>* terms;
  uint32_t* offs;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    in = c.take<uint8_t>(kPair * n); terms = c.take<XYZZ<F>>(n); pst = c.take<uint8_t>(n); offs = c.take<uint32_t>(count + 1);
    dout = c.take<uint8_t>(kPt * count); dst = c.take<uint8_t>(count);
  }));
  if (n) {
    B2_CUDA(ctx, cudaMemcpyAsync(in, pairs, kPair * n, cudaMemcpyHostToDevice, st));
    B2_LAUNCH(ctx, bls_msm_terms<F>, (unsigned)((n + 63) / 64), 64, 0, st, (const uint8_t*)in, n, terms, pst);
  }
  B2_CUDA(ctx, cudaMemcpyAsync(offs, pair_offsets, (count + 1) * 4, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, bls_msm_fold<F>, (unsigned)count, kFoldThreads, 0, st, (const XYZZ<F>*)terms, (const uint8_t*)pst, (const uint32_t*)offs, dout, dst);
  B2_CUDA(ctx, cudaMemcpyAsync(out, dout, kPt * count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(status, dst, count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

}  // namespace
}  // namespace b200zk

using namespace b200zk;

extern "C" {

int b200zk_bls12_381_g1_add_batch(b200zk_ctx* ctx, const uint8_t* a, const uint8_t* b, size_t count, uint8_t* out, uint8_t* status) {
  return add_batch<Fp381>(ctx, "bls12_381_g1_add_batch", a, b, count, out, status);
}

int b200zk_bls12_381_g2_add_batch(b200zk_ctx* ctx, const uint8_t* a, const uint8_t* b, size_t count, uint8_t* out, uint8_t* status) {
  return add_batch<F2>(ctx, "bls12_381_g2_add_batch", a, b, count, out, status);
}

int b200zk_bls12_381_g1_msm_batch(b200zk_ctx* ctx, const uint8_t* pairs, const uint32_t* pair_offsets, size_t count, uint8_t* out, uint8_t* status) {
  return msm_batch<Fp381>(ctx, "bls12_381_g1_msm_batch", pairs, pair_offsets, count, out, status);
}

int b200zk_bls12_381_g2_msm_batch(b200zk_ctx* ctx, const uint8_t* pairs, const uint32_t* pair_offsets, size_t count, uint8_t* out, uint8_t* status) {
  return msm_batch<F2>(ctx, "bls12_381_g2_msm_batch", pairs, pair_offsets, count, out, status);
}

}  // extern "C"
