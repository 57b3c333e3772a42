// bls381.cu -- BLS12-381 G1 byte formats on the device and the EIP-4844 blob commitment entry points
// (SURVEY.md section 8f row 3):
//   /root/reference/crates/common/crypto/kzg.rs:259-272        blob_to_kzg_commitment_and_proof -> c_kzg blob_to_kzg_commitment
//   /root/reference/crates/common/types/blobs_bundle.rs:90-118 BlobsBundle::create_from_blobs (one commitment per blob)
// A blob is 4096 field elements (32-byte big-endian, each < the BLS12-381 group order r); its commitment is
// sum_i blob[i] * L_i over the trusted setup's 4096 G1 points in Lagrange form (bit-reversed order, as c-kzg stores them),
// returned in the 48-byte compressed format.  The MSM itself is msm.cu instantiated over Fp381 (window tables included).
// The proof (c-kzg compute_kzg_proof / compute_blob_kzg_proof) evaluates p at z and builds the quotient on the device
// (kzg_eval_quotient, over the scalar field Fr381), then commits to it with the same MSM.
#include "bls12.cuh"
#include "cell_batch.h"
#include "sha256.h"
#include <cstring>
#include <vector>

namespace b200zk {

// status[0] = first index whose coordinate is >= p, status[1] = first index that is not a curve point or whose flag bits
// are inconsistent (atomicMin; initialised to n by the host)
__global__ void __launch_bounds__(64) bls_g1_decode(const uint8_t* __restrict__ in, void* __restrict__ native, size_t n, int compressed, unsigned long long* status) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* src = in + i * (compressed ? 48 : 96);
  const uint8_t flags = src[0];
  const bool c_flag = flags & 0x80, inf_flag = flags & 0x40, sign_flag = flags & 0x20;
  Affine<Fp381> pt = {Fp381::zero(), Fp381::zero()};
  bool bad_field = false, bad_point = false;
  if (compressed) {
    const uint32_t st = bls_g1_decompress(src, &pt);
    bad_field = st == B200ZK_ERR_NOT_IN_FIELD;
    bad_point = st == B200ZK_ERR_NOT_ON_CURVE;
  } else {  // uncompressed: x | y big-endian, flag bits must be clear except infinity
    const Fp381 x = load_be48(src, 0x1fffffffu);
    Fp381 y = load_be48(src + 48, 0xffffffffu);
    if (c_flag || sign_flag) bad_point = true;
    else if (inf_flag) { if (!x.is_zero() || !y.is_zero()) bad_point = true; }
    else if (!Fp381::less(x, Fp381::modulus()) || !Fp381::less(y, Fp381::modulus())) bad_field = true;
    else {
      pt = {Fp381::to_mont(x), Fp381::to_mont(y)};
      if (pt.is_inf() || !affine_on_curve(pt)) bad_point = true;
    }
  }
  if (bad_field) atomicMin(status, (unsigned long long)i);
  if (bad_point) atomicMin(status + 1, (unsigned long long)i);
  if (bad_field || bad_point) pt = {Fp381::zero(), Fp381::zero()};
  store_affine<Fp381>(native, i, pt);
}

// first index of a 32-byte scalar (big-endian, or little-endian limbs) that is not below the BLS12-381 group order
__global__ void __launch_bounds__(256) bls_scalar_check(const uint8_t* __restrict__ scalars, size_t n, int big_endian, unsigned long long* bad) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(scalars + 32 * i);
  uint64_t br = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint32_t limb = big_endian ? __byte_perm(__ldg(w + 7 - k), 0, 0x0123) : __ldg(w + k);
    const uint64_t d = (uint64_t)limb - bls_r_limb(k) - br;
    br = (d >> 32) & 1u;
  }
  if (!br) atomicMin(bad, (unsigned long long)i);  // no borrow: scalar >= r
}

// ---- EIP-4844 proofs: p(z) and the quotient (p(X) - p(z)) / (X - z) of a blob in evaluation form -------------------
constexpr uint32_t kBlobN = 4096;      // FIELD_ELEMENTS_PER_BLOB
constexpr uint32_t kEvalThreads = 256;  // one CTA per blob, 16 elements per thread: element k * 256 + t belongs to thread t
constexpr size_t kEvalSmem = (kBlobN + 2 * kEvalThreads) * 32;  // per-element products / inverses + a 512-node product tree

// roots[i] = w^brp(i), i < 4096, w = 7^((r-1)/4096) (c-kzg's g1_lagrange_brp order); roots[4096] = 1/4096 = r - (r-1)/4096.
// Montgomery form.  One thread per entry, each deriving w from its definition: a one-off per context.
__global__ void __launch_bounds__(256) kzg_roots_build(void* __restrict__ roots) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > kBlobN) return;
  Fr381 e;  // (r - 1) / 4096 = (r - 1) >> 12 (r - 1 = r with limb 0 cleared)
#pragma unroll
  for (int k = 0; k < 8; ++k) e.v[k] = ((k ? bls_r_limb(k) : 0u) >> 12) | (k < 7 ? bls_r_limb(k + 1) << 20 : 0u);
  if (i == kBlobN) { store_fe(roots, i, Fr381::to_mont(Fr381::sub(Fr381::zero(), e))); return; }
  Fr381 c = Fr381::zero();
  c.v[0] = 7;
  Fr381 base = Fr381::pow(Fr381::to_mont(c), e.v), acc = Fr381::one();
#pragma unroll 1
  for (uint32_t x = __brev(i) >> 20; x; x >>= 1) {  // w^brp(i), square and multiply over the 12-bit exponent
    if (x & 1) acc = Fr381::mul(acc, base);
    base = Fr381::sqr(base);
  }
  store_fe(roots, i, acc);
}

// d_i = z - w_i, except where z = w_m: there the batch inverts z instead of 0, so slot m yields z^-1
B2_D Fr381 eval_denominator(const Fr381& z, const void* roots, uint32_t i, uint32_t* s_m) {
  const Fr381 d = Fr381::sub(z, load_fe_nc<Fr381>(roots, i));
  if (!d.is_zero()) return d;
  *s_m = i;
  return z;
}

// One CTA per blob.  In: the blobs (4096 x 32-byte big-endian, already checked < r), z (32-byte big-endian, < r), the root
// table.  Out: y = p(z) (32-byte big-endian) and the quotient q as canonical little-endian limbs, the proof MSM's scalars.
//   z outside the domain: y = (z^4096 - 1)/4096 * sum_i p_i w_i / (z - w_i),  q_i = (y - p_i) / (z - w_i)
//   z = w_m:             y = p_m,  q_i as above for i != m,  q_m = sum_{i != m} (p_i - y) w_i / (z (z - w_i)) = -z^-1 sum_{i != m} q_i w_i
// All 4096 inverses come from one Montgomery batch: per-thread prefix products, a product tree over the 256 threads, one
// Fermat inversion at its root.  p_i and y stay canonical: mul(canonical, Montgomery) is the canonical product, so
// neither the inputs nor the quotient need a conversion.
__global__ void __launch_bounds__(kEvalThreads, 1) kzg_eval_quotient(const uint8_t* __restrict__ blobs, const uint8_t* __restrict__ z_be, const void* __restrict__ roots,
                                                                    void* __restrict__ q_out, uint8_t* __restrict__ y_be) {
  extern __shared__ uint4 kzg_smem[];
  uint4* pre = kzg_smem;                 // 4096 elements: prefix products, then the inverses d_i^-1
  uint4* tree = kzg_smem + 2 * kBlobN;   // 512 nodes: 1 = root, 256 + t = thread t's product; later a reduction buffer
  __shared__ uint32_t s_m;
  const uint32_t t = threadIdx.x;
  const uint8_t* blob = blobs + (size_t)blockIdx.x * kBlobN * 32;
  void* q = (uint8_t*)q_out + (size_t)blockIdx.x * kBlobN * 32;
  if (t == 0) s_m = kBlobN;
  const Fr381 z = Fr381::to_mont(load_be32(z_be + 32 * blockIdx.x));
  __syncthreads();
  Fr381 acc = Fr381::one();
#pragma unroll 1
  for (uint32_t k = 0; k < kBlobN / kEvalThreads; ++k) {
    const uint32_t i = k * kEvalThreads + t;
    acc = Fr381::mul(acc, eval_denominator(z, roots, i, &s_m));
    store_fe(pre, i, acc);
  }
  store_fe(tree, kEvalThreads + t, acc);
  __syncthreads();
  for (uint32_t lvl = kEvalThreads / 2; lvl >= 1; lvl >>= 1) {
    if (t < lvl) store_fe(tree, lvl + t, Fr381::mul(load_fe<Fr381>(tree, 2 * (lvl + t)), load_fe<Fr381>(tree, 2 * (lvl + t) + 1)));
    __syncthreads();
  }
  if (t == 0) store_fe(tree, 1, Fr381::inv(load_fe<Fr381>(tree, 1)));
  __syncthreads();
  for (uint32_t lvl = 1; lvl < kEvalThreads; lvl <<= 1) {  // node j holds (its product)^-1: hand each child the other's product
    if (t < lvl) {
      const uint32_t j = lvl + t;
      const Fr381 x = load_fe<Fr381>(tree, j), a = load_fe<Fr381>(tree, 2 * j), b = load_fe<Fr381>(tree, 2 * j + 1);
      store_fe(tree, 2 * j, Fr381::mul(x, b));
      store_fe(tree, 2 * j + 1, Fr381::mul(x, a));
    }
    __syncthreads();
  }
  const uint32_t m = s_m;
  Fr381 inv_acc = load_fe<Fr381>(tree, kEvalThreads + t), s = Fr381::zero();
#pragma unroll 1
  for (int k = kBlobN / kEvalThreads - 1; k >= 0; --k) {
    const uint32_t i = k * kEvalThreads + t;
    const Fr381 w = load_fe_nc<Fr381>(roots, i);
    const Fr381 di = k ? Fr381::mul(inv_acc, load_fe<Fr381>(pre, i - kEvalThreads)) : inv_acc;
    inv_acc = Fr381::mul(inv_acc, i == m ? z : Fr381::sub(z, w));
    store_fe(pre, i, di);
    if (i != m) s = Fr381::add(s, Fr381::mul(Fr381::mul(load_be32(blob + 32 * i), w), di));
  }
  store_fe(tree, t, s);  // nodes 0..255: free since the down-sweep
  __syncthreads();
  for (uint32_t h = kEvalThreads / 2; h >= 1; h >>= 1) {
    if (t < h) store_fe(tree, t, Fr381::add(load_fe<Fr381>(tree, t), load_fe<Fr381>(tree, t + h)));
    __syncthreads();
  }
  if (t == 0) {
    Fr381 y;
    if (m < kBlobN) y = load_be32(blob + 32 * m);
    else {
      Fr381 zn = z;
      for (int k = 0; k < 12; ++k) zn = Fr381::sqr(zn);  // z^4096
      y = Fr381::mul(Fr381::mul(Fr381::sub(zn, Fr381::one()), load_fe_nc<Fr381>(roots, kBlobN)), load_fe<Fr381>(tree, 0));
    }
    store_fe(tree, 0, y);
    store_be32(y_be + 32 * blockIdx.x, y);
  }
  __syncthreads();
  const Fr381 y = load_fe<Fr381>(tree, 0);
  Fr381 tq = Fr381::zero();
#pragma unroll 1
  for (uint32_t k = 0; k < kBlobN / kEvalThreads; ++k) {
    const uint32_t i = k * kEvalThreads + t;
    if (i == m) continue;
    const Fr381 qi = Fr381::mul(Fr381::sub(y, load_be32(blob + 32 * i)), load_fe<Fr381>(pre, i));
    store_fe(q, i, qi);
    if (m < kBlobN) tq = Fr381::add(tq, Fr381::mul(qi, load_fe_nc<Fr381>(roots, i)));
  }
  if (m < kBlobN) {  // the same branch in every thread
    __syncthreads();   // everyone has read y out of node 0
    store_fe(tree, t, tq);
    __syncthreads();
    for (uint32_t h = kEvalThreads / 2; h >= 1; h >>= 1) {
      if (t < h) store_fe(tree, t, Fr381::add(load_fe<Fr381>(tree, t), load_fe<Fr381>(tree, t + h)));
      __syncthreads();
    }
    if (t == 0) store_fe(q, m, Fr381::neg(Fr381::mul(load_fe<Fr381>(tree, 0), load_fe<Fr381>(pre, m))));  // pre[m] = z^-1
  }
}

int bls_points_to_native(b200zk_ctx* ctx, const void* d_in, void* d_native, size_t n, bool compressed, cudaStream_t st) {
  if (!n) return B200ZK_OK;
  B2_TRY(ensure(ctx, ctx->ws_misc, 512));
  unsigned long long* status = (unsigned long long*)((uint8_t*)ctx->ws_misc.p + 256);
  unsigned long long* h = (unsigned long long*)(ctx->h_pinned + 1024);
  h[0] = h[1] = (unsigned long long)n;
  B2_CUDA(ctx, cudaMemcpyAsync(status, h, 16, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, bls_g1_decode, (unsigned)((n + 63) / 64), 64, 0, st, (const uint8_t*)d_in, d_native, n, compressed ? 1 : 0, status);
  B2_CUDA(ctx, cudaMemcpyAsync(h, status, 16, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (h[0] < n && h[0] <= h[1]) return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, "bls12-381 point: coordinate >= p");
  if (h[1] < n) return fail(ctx, B200ZK_ERR_NOT_ON_CURVE, "bls12-381 point: not on the curve or malformed flag bits");
  return B200ZK_OK;
}

int bls_scalars_check(b200zk_ctx* ctx, const void* d_scalars, size_t n, bool big_endian, cudaStream_t st, size_t* bad_index) {
  *bad_index = n;
  if (!n) return B200ZK_OK;
  B2_TRY(ensure(ctx, ctx->ws_misc, 512));
  unsigned long long* status = (unsigned long long*)((uint8_t*)ctx->ws_misc.p + 256);
  unsigned long long* h = (unsigned long long*)(ctx->h_pinned + 1024);
  h[0] = (unsigned long long)n;
  B2_CUDA(ctx, cudaMemcpyAsync(status, h, 8, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, bls_scalar_check, (unsigned)((n + 255) / 256), 256, 0, st, (const uint8_t*)d_scalars, n, big_endian ? 1 : 0, status);
  B2_CUDA(ctx, cudaMemcpyAsync(h, status, 8, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  *bad_index = (size_t)h[0];
  return B200ZK_OK;
}

int bls_scalars_check_enqueue(b200zk_ctx* ctx, const void* d_scalars, size_t n, bool big_endian, cudaStream_t st, unsigned long long* d_bad) {
  if (n) B2_LAUNCH(ctx, bls_scalar_check, (unsigned)((n + 255) / 256), 256, 0, st, (const uint8_t*)d_scalars, n, big_endian ? 1 : 0, d_bad);
  return B200ZK_OK;
}

}  // namespace b200zk

using namespace b200zk;

namespace {
int bls_msm_host_scalars(b200zk_ctx* ctx, const BasesEntry& e, const void* scalars, size_t n, uint32_t flags, cudaStream_t st, uint8_t out[48]) {
  // scalars must be canonical field elements of the BLS12-381 scalar field (c-kzg bytes_to_bls_field rejects the rest), in
  // either byte order: the MSM does not reduce them, and a value >= 2^255 would overflow the signed-digit recoding's top window
  B2_TRY(ensure(ctx, ctx->ws_scalars, n * 32 + 32));
  if (n) B2_CUDA(ctx, cudaMemcpyAsync(ctx->ws_scalars.p, scalars, n * 32, cudaMemcpyHostToDevice, st));
  size_t bad = n;
  B2_TRY(bls_scalars_check(ctx, ctx->ws_scalars.p, n, (flags & B200ZK_SCALARS_BE) != 0, st, &bad));
  if (bad < n) return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, "bls12-381 scalar >= the group order");
  B2_TRY(ensure(ctx, ctx->ws_result, 512));
  B2_TRY(ensure(ctx, ctx->ws_out, 512));
  B2_TRY(msm_run_bls(ctx, e.d.p, ctx->ws_scalars.p, n, flags & (B200ZK_SCALARS_BE | B200ZK_SCALARS_RAW), st, ctx->ws_result.p, e.table_c, e.n));
  B2_TRY(msm_encode_bls(ctx, ctx->ws_result.p, 1, flags, st, ctx->ws_out.p));
  B2_CUDA(ctx, cudaMemcpyAsync(ctx->h_pinned, ctx->ws_out.p, 96 + 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  memcpy(out, ctx->h_pinned, 48);
  uint32_t inf;
  memcpy(&inf, ctx->h_pinned + 96, 4);
  return inf ? B200ZK_OK_INFINITY : B200ZK_OK;
}

// the root table (kzg_roots_build), built on first use
int kzg_roots(b200zk_ctx* ctx, cudaStream_t st, const void** roots) {
  return once_table(ctx, ctx->kzg_roots, (kBlobN + 1) * 32, st, [&](void* t) -> int {
    B2_LAUNCH(ctx, kzg_roots_build, (kBlobN + 256) / 256, 256, 0, st, t);
    return B200ZK_OK;
  }, roots);
}

// ws_kzg for n blobs: [blobs n x 128 KiB, then z n x 32 right behind them (one range check covers both) | quotients
// n x 128 KiB | y n x 32 | 2n XYZZ partial sums | 2n encoded points (commitments, then proofs)]
struct KzgLayout {
  uint8_t *blobs, *z, *q, *y, *partials, *enc;
  static constexpr size_t kPartial = 4 * 48, kEnc = 128;  // msm_encode writes 96 B + a u32 is_infinity flag
  int make(b200zk_ctx* ctx, size_t n) {
    B2_TRY(carve(ctx, ctx->ws_kzg, [&](Carve& c) {
      blobs = c.take<uint8_t>(n * (kBlobN + 1) * 32); q = c.take<uint8_t>(n * kBlobN * 32); y = c.take<uint8_t>(n * 32);
      partials = c.take<uint8_t>(2 * n * kPartial); enc = c.take<uint8_t>(2 * n * kEnc);
    }));
    z = blobs + n * kBlobN * 32;
    return B200ZK_OK;
  }
};

}  // namespace

// one 4096-point MSM per blob over the setup, each encoded into its own 128-byte slot of `enc`
int b200zk::kzg_msms(b200zk_ctx* ctx, const BasesEntry& e, const uint8_t* scalars, size_t n, uint32_t flags, uint8_t* partials, uint8_t* enc, cudaStream_t st) {
  for (size_t b = 0; b < n; ++b) {
    B2_TRY(msm_run_bls(ctx, e.d.p, scalars + b * kBlobN * 32, kBlobN, flags, st, partials + b * KzgLayout::kPartial, e.table_c, e.n));
    B2_TRY(msm_encode_bls(ctx, partials + b * KzgLayout::kPartial, 1, 0, st, enc + b * KzgLayout::kEnc));
  }
  return B200ZK_OK;
}

// the setup handle of a KZG call: a BLS12-381 G1 handle of exactly 4096 points
int b200zk::kzg_setup(b200zk_ctx* ctx, uint64_t handle, const char* what, BasesEntry** e) {
  std::string msg = what;
  *e = find_bases(ctx, handle, Group::Bls12G1, (msg + ": unknown setup handle").c_str());
  if (!*e) return B200ZK_ERR_INVALID_ARG;
  if ((*e)->n != kBlobN) return fail(ctx, B200ZK_ERR_INVALID_ARG, (msg + ": the setup must hold FIELD_ELEMENTS_PER_BLOB = 4096 points").c_str());
  return B200ZK_OK;
}

namespace {
// z of every blob in L.z, checked: y into L.y, the proofs' encodings into enc
int kzg_proofs(b200zk_ctx* ctx, const BasesEntry& e, const KzgLayout& L, size_t n, uint8_t* enc, cudaStream_t st) {
  B2_TRY(kzg_eval_run(ctx, L.blobs, L.z, n, L.q, L.y, st));
  return kzg_msms(ctx, e, L.q, n, 0 /* little-endian limbs */, L.partials + n * KzgLayout::kPartial, enc, st);
}
}  // namespace

// EIP-4844 compute_challenge: hash_to_bls_field(SHA-256("FSBLOBVERIFY_V1_" | 4096 as 16-byte big-endian | blob | commitment))
void b200zk::kzg_challenge(const uint8_t* blob, const uint8_t commitment[48], uint8_t z_be[32]) {
  static const uint8_t kDomain[16] = {'F', 'S', 'B', 'L', 'O', 'B', 'V', 'E', 'R', 'I', 'F', 'Y', '_', 'V', '1', '_'};
  uint8_t degree[16] = {};
  degree[14] = kBlobN >> 8;
  Sha256 h;
  h.update(kDomain, 16);
  h.update(degree, 16);
  h.update(blob, kBlobN * 32);
  h.update(commitment, 48);
  uint8_t d[32];
  h.final(d);
  hash_to_bls_field(d, z_be);
}

// y = p(z) of n blobs (kzg_eval_quotient, one CTA per blob); the quotient goes to q (n x 4096 x 32 bytes)
int b200zk::kzg_eval_run(b200zk_ctx* ctx, const uint8_t* d_blobs, const uint8_t* d_z, size_t n, void* d_q, uint8_t* d_y, cudaStream_t st) {
  const void* roots = nullptr;
  B2_TRY(kzg_roots(ctx, st, &roots));
  if (!ctx->attr_kzg) {
    B2_CUDA(ctx, cudaFuncSetAttribute(kzg_eval_quotient, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kEvalSmem));
    ctx->attr_kzg = true;
  }
  B2_LAUNCH(ctx, kzg_eval_quotient, (unsigned)n, kEvalThreads, kEvalSmem, st, d_blobs, d_z, roots, d_q, d_y);
  return B200ZK_OK;
}

extern "C" {

int b200zk_bls12_381_g1_bases_upload(b200zk_ctx* ctx, const void* points, size_t n, uint32_t flags, uint64_t* handle) {
  if (!ctx || !handle || (!points && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bls12_381_g1_bases_upload: null argument");
  DeviceGuard guard(ctx);
  const bool compressed = flags & B200ZK_POINTS_COMPRESSED;
  const size_t in_bytes = n * (compressed ? 48 : 96);
  BasesEntry e;
  e.n = n; e.group = Group::Bls12G1;
  B2_CUDA(ctx, cudaMalloc(&e.d.p, n * 96 + 32));
  int rc = ensure(ctx, ctx->ws_ntt, in_bytes + 32);
  cudaError_t ce = cudaSuccess;
  if (rc <= B200ZK_OK_INFINITY && n) ce = cudaMemcpyAsync(ctx->ws_ntt.p, points, in_bytes, cudaMemcpyHostToDevice, ctx->stream);
  if (rc <= B200ZK_OK_INFINITY && ce == cudaSuccess) rc = bls_points_to_native(ctx, ctx->ws_ntt.p, e.d.p, n, compressed, ctx->stream);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(ctx->stream);
  if (rc > B200ZK_OK_INFINITY) return rc;
  if (ce != cudaSuccess) return fail(ctx, B200ZK_ERR_CUDA, "bls bases upload", ce);
  return register_bases(ctx, std::move(e), handle);
}

int b200zk_bls12_381_g1_msm_resident(b200zk_ctx* ctx, uint64_t handle, const void* scalars, size_t n, uint32_t flags, uint8_t out[48]) {
  if (!ctx || !out || (!scalars && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bls12_381_g1_msm_resident: null argument");
  DeviceGuard guard(ctx);
  const BasesEntry* e = find_bases(ctx, handle, Group::Bls12G1, "bls12_381_g1_msm_resident: unknown handle");
  if (!e) return B200ZK_ERR_INVALID_ARG;
  if (n > e->n) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bls12_381_g1_msm_resident: n exceeds the resident bases");
  return bls_msm_host_scalars(ctx, *e, scalars, n, flags, ctx->stream, out);
}

int b200zk_kzg_blob_to_commitment(b200zk_ctx* ctx, uint64_t setup_handle, const uint8_t* blobs, size_t n_blobs, uint8_t* commitments) {
  if (!ctx || (n_blobs && (!blobs || !commitments))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_blob_to_commitment: null argument");
  DeviceGuard guard(ctx);
  BasesEntry* e = nullptr;
  B2_TRY(kzg_setup(ctx, setup_handle, "kzg_blob_to_commitment", &e));
  for (size_t b = 0; b < n_blobs; ++b) {
    int rc = bls_msm_host_scalars(ctx, *e, blobs + b * 4096 * 32, 4096, B200ZK_SCALARS_BE | B200ZK_SCALARS_RAW, ctx->stream, commitments + 48 * b);
    if (rc > B200ZK_OK_INFINITY) return rc;
  }
  return B200ZK_OK;
}

int b200zk_kzg_blob_to_commitment_and_proof(b200zk_ctx* ctx, uint64_t setup_handle, const uint8_t* blobs, size_t n_blobs, uint8_t* commitments, uint8_t* proofs) {
  static const char* what = "kzg_blob_to_commitment_and_proof";
  if (!ctx || (n_blobs && (!blobs || !commitments || !proofs))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_blob_to_commitment_and_proof: null argument");
  NvtxRange nvtx("b200zk:kzg_blob_to_commitment_and_proof");
  DeviceGuard guard(ctx);
  BasesEntry* e = nullptr;
  B2_TRY(kzg_setup(ctx, setup_handle, what, &e));
  if (!n_blobs) return B200ZK_OK;
  cudaStream_t st = ctx->stream;
  KzgLayout L;
  B2_TRY(L.make(ctx, n_blobs));
  B2_CUDA(ctx, cudaMemcpyAsync(L.blobs, blobs, n_blobs * kBlobN * 32, cudaMemcpyHostToDevice, st));
  B2_TRY(check_blobs(ctx, L.blobs, n_blobs, 0, st, what));
  // commitments, read back once: the challenge hashes them on the host
  B2_TRY(kzg_msms(ctx, *e, L.blobs, n_blobs, B200ZK_SCALARS_BE, L.partials, L.enc, st));
  std::vector<uint8_t> enc(2 * n_blobs * KzgLayout::kEnc), z(n_blobs * 32);
  B2_CUDA(ctx, cudaMemcpyAsync(enc.data(), L.enc, n_blobs * KzgLayout::kEnc, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  for (size_t b = 0; b < n_blobs; ++b) kzg_challenge(blobs + b * kBlobN * 32, &enc[b * KzgLayout::kEnc], &z[32 * b]);
  B2_CUDA(ctx, cudaMemcpyAsync(L.z, z.data(), n_blobs * 32, cudaMemcpyHostToDevice, st));
  uint8_t* enc_proofs = L.enc + n_blobs * KzgLayout::kEnc;
  B2_TRY(kzg_proofs(ctx, *e, L, n_blobs, enc_proofs, st));
  B2_CUDA(ctx, cudaMemcpyAsync(enc.data() + n_blobs * KzgLayout::kEnc, enc_proofs, n_blobs * KzgLayout::kEnc, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  for (size_t b = 0; b < n_blobs; ++b) {
    memcpy(commitments + 48 * b, &enc[b * KzgLayout::kEnc], 48);
    memcpy(proofs + 48 * b, &enc[(n_blobs + b) * KzgLayout::kEnc], 48);
  }
  return B200ZK_OK;
}

int b200zk_kzg_compute_proof(b200zk_ctx* ctx, uint64_t setup_handle, const uint8_t* blobs, size_t n_blobs, const uint8_t* z, uint8_t* proofs, uint8_t* y) {
  static const char* what = "kzg_compute_proof";
  if (!ctx || (n_blobs && (!blobs || !z || !proofs || !y))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_compute_proof: null argument");
  NvtxRange nvtx("b200zk:kzg_compute_proof");
  DeviceGuard guard(ctx);
  BasesEntry* e = nullptr;
  B2_TRY(kzg_setup(ctx, setup_handle, what, &e));
  if (!n_blobs) return B200ZK_OK;
  cudaStream_t st = ctx->stream;
  KzgLayout L;
  B2_TRY(L.make(ctx, n_blobs));
  B2_CUDA(ctx, cudaMemcpyAsync(L.blobs, blobs, n_blobs * kBlobN * 32, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(L.z, z, n_blobs * 32, cudaMemcpyHostToDevice, st));
  B2_TRY(check_blobs(ctx, L.blobs, n_blobs, n_blobs, st, what));
  B2_TRY(kzg_proofs(ctx, *e, L, n_blobs, L.enc, st));
  std::vector<uint8_t> enc(n_blobs * KzgLayout::kEnc), ys(n_blobs * 32);
  B2_CUDA(ctx, cudaMemcpyAsync(enc.data(), L.enc, enc.size(), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(ys.data(), L.y, ys.size(), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  for (size_t b = 0; b < n_blobs; ++b) memcpy(proofs + 48 * b, &enc[b * KzgLayout::kEnc], 48);
  memcpy(y, ys.data(), ys.size());
  return B200ZK_OK;
}

}  // extern "C"
