// groth16_verify.cu -- Groth16 batch verification on the device (b200zk_groth16_verify_batch): N proofs against one
// verifying key with one pairing product.  With independent 128-bit coefficients rho_i the N equations
//   e(A_i, B_i) = e(alpha, beta) e(vk_x(i), gamma) e(C_i, delta),   vk_x(i) = IC_0 + sum_j x_ij IC_j
// hold together (up to probability 2^-128) exactly when
//   prod_i e(-rho_i A_i, B_i) * e(s_0 alpha, beta) * e(sum_j s_j IC_j, gamma) * e(sum_i rho_i C_i, delta) = 1,
//   s_0 = sum_i rho_i, s_j = sum_i rho_i x_ij
// holds: N + 3 Miller loops and one final exponentiation.  DESIGN.md section 4.20 has the soundness argument.  When the
// combined check fails, every well-formed proof is decided by its own 4-pair check on the device.  One stream; the host
// hashes the inputs into the coefficients while the device decodes them.
#include <algorithm>
#include <cstring>

#include "bn_pairing.cuh"
#include "sha256.h"

namespace b200zk {
namespace {

constexpr unsigned kSumThreads = 128;   // XYZZ<Fq> tree sums: 128 B of shared memory per thread
constexpr unsigned kSumBlocks = 64;
constexpr unsigned kProdThreads = 32;   // Fq12 tree products: 384 B per thread
constexpr unsigned kProdBlocks = 128;
constexpr unsigned kScalarThreads = 256;
constexpr size_t kMaxCount = (size_t)1 << 28;  // 4 count + 3 pairs index with 32 bits

B2_D Affine<Fq> g1_identity() { return {Fq::zero(), Fq::zero()}; }
B2_D Affine<Fq> g1_neg(const Affine<Fq>& p) { return {p.x, Fq::neg(p.y)}; }  // neg(0) = 0: the identity stays (0, 0)

// rho_i: 16 big-endian bytes as the low four limbs of a 256-bit little-endian scalar
B2_D void load_rho(const uint8_t* rho_be, size_t i, uint32_t k[8]) {
#pragma unroll
  for (int j = 0; j < 8; ++j) k[j] = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const uint8_t* b = rho_be + 16 * i + 4 * (3 - j);
    k[j] = ((uint32_t)b[0] << 24) | ((uint32_t)b[1] << 16) | ((uint32_t)b[2] << 8) | (uint32_t)b[3];
  }
}

// One thread per verifying-key element e: 0 alpha1, 1..3 beta2, gamma2, delta2 (each in the order-r subgroup), 4 + j
// IC_j.  g1 = alpha1 | IC_0 .. IC_n_pub, g2 = beta2 | gamma2 | delta2; vst[e] = 0, 2 or 3.
__global__ void __launch_bounds__(64) g16v_vk_decode(const uint8_t* vk, uint32_t n_ic, Affine<Fq>* g1, Affine<Fq2>* g2, uint8_t* vst) {
  const size_t e = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (e >= 4 + (size_t)n_ic) return;
  uint32_t s;
  if (e == 0 || e >= 4) {
    Affine<Fq> p = g1_identity();
    s = decode_g1(vk + (e == 0 ? 0 : 448 + 64 * (e - 4)), &p);
    g1[e == 0 ? 0 : e - 3] = p;
  } else {
    Affine<Fq2> q = {Fq2::zero(), Fq2::zero()};
    s = decode_g2(vk + 64 + 128 * (e - 1), &q);
    if (!s && !q.is_inf() && !in_subgroup<FrCfg::mod>(q)) s = B200ZK_ERR_NOT_ON_CURVE;
    g2[e - 1] = q;
  }
  vst[e] = (uint8_t)s;
}

// One thread per proof: A | B | C and the proof's public inputs with the precompile's error order (every coordinate < p
// and every input < r before any curve check), B in the order-r subgroup.  st[i] = 0, 2 or 3.
__global__ void __launch_bounds__(64) g16v_decode(const uint8_t* proofs, const uint8_t* x, uint32_t n_pub, size_t n, Affine<Fq>* A, Affine<Fq2>* B,
                                                  Affine<Fq>* C, uint8_t* st) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* pr = proofs + 256 * i;
  Affine<Fq> a = g1_identity(), c = g1_identity();
  Affine<Fq2> b = {Fq2::zero(), Fq2::zero()};
  const uint32_t sa = decode_g1(pr, &a), sb = decode_g2(pr + 64, &b), sc = decode_g1(pr + 192, &c);
  bool x_ok = true;
  for (uint32_t j = 0; j < n_pub; ++j) {
    bool ok;
    load_be<Fr>(x + 32 * (i * n_pub + j), &ok);
    x_ok = x_ok && ok;
  }
  uint32_t s = (!x_ok || sa == B200ZK_ERR_NOT_IN_FIELD || sb == B200ZK_ERR_NOT_IN_FIELD || sc == B200ZK_ERR_NOT_IN_FIELD)
                   ? (uint32_t)B200ZK_ERR_NOT_IN_FIELD : (sa ? sa : (sb ? sb : sc));
  if (!s && !b.is_inf() && !in_subgroup<FrCfg::mod>(b)) s = B200ZK_ERR_NOT_ON_CURVE;
  A[i] = a;
  B[i] = b;
  C[i] = c;
  st[i] = (uint8_t)s;
}

// One thread per proof, a malformed one (st != 0) left out: P[i] = -rho_i A_i (affine, paired with B_i), T[i] = rho_i C_i.
// rho_i has 128 bits, so the double-and-add walks 128.
__global__ void __launch_bounds__(64) g16v_terms(const uint8_t* rho_be, const uint8_t* st, const Affine<Fq>* A, const Affine<Fq>* C, size_t n,
                                                 Affine<Fq>* P, XYZZ<Fq>* T) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (st[i]) { P[i] = g1_identity(); T[i] = XYZZ<Fq>::identity(); return; }
  uint32_t k[8];
  load_rho(rho_be, i, k);
  P[i] = g1_neg(xyzz_to_affine(xyzz_scalar_mul<Fq>(k, A[i], 128)));
  T[i] = xyzz_scalar_mul<Fq>(k, C[i], 128);
}

// s_j = sum_i rho_i x_ij over the well-formed proofs (x_i0 = 1), one CTA per j: a strided share per thread, then a tree in
// shared memory.  mul(canonical rho, Montgomery x) is the canonical product, so s is canonical.
__global__ void __launch_bounds__(kScalarThreads) g16v_scalars(const uint8_t* rho_be, const uint8_t* st, const uint8_t* x, uint32_t n_pub, size_t n, Fr* s) {
  __shared__ Fr sh[kScalarThreads];
  const uint32_t j = blockIdx.x, t = threadIdx.x;
  Fr acc = Fr::zero();
  for (size_t i = t; i < n; i += kScalarThreads) {
    if (st[i]) continue;
    Fr r;
    load_rho(rho_be, i, r.v);
    if (j == 0) {
      acc = Fr::add(acc, r);
    } else {
      bool ok;
      acc = Fr::add(acc, Fr::mul(r, Fr::to_mont(load_be<Fr>(x + 32 * (i * n_pub + j - 1), &ok))));
    }
  }
  sh[t] = acc;
  __syncthreads();
  for (uint32_t w = kScalarThreads / 2; w; w >>= 1) {
    if (t < w) sh[t] = Fr::add(sh[t], sh[t + w]);
    __syncthreads();
  }
  if (!t) s[j] = sh[0];
}

// One thread per IC point and one for alpha1: T[j] = s_j IC_j (j < n_ic), *P_alpha = s_0 alpha1 (affine)
__global__ void __launch_bounds__(64) g16v_vk_terms(const Fr* s, const Affine<Fq>* g1, uint32_t n_ic, XYZZ<Fq>* T, Affine<Fq>* P_alpha) {
  const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (t > n_ic) return;
  const Fr k = s[t < n_ic ? t : 0];
  if (t < n_ic) T[t] = xyzz_scalar_mul<Fq>(k.v, g1[1 + t]);
  else *P_alpha = xyzz_to_affine(xyzz_scalar_mul<Fq>(k.v, g1[0]));
}

// Tree sum of XYZZ terms, segment y = blockIdx.y over T[lo[y], hi[y]): every thread adds a grid-strided share, then a tree
// in shared memory.  Several CTAs write partial[y gridDim.x + blockIdx.x]; one CTA (the second launch over those partials)
// writes the affine sum to out[y].
struct Segs { size_t lo[2], hi[2]; };
__global__ void __launch_bounds__(kSumThreads) g16v_sum(const XYZZ<Fq>* T, Segs sg, XYZZ<Fq>* partial, Affine<Fq>* out) {
  __shared__ XYZZ<Fq> sh[kSumThreads];
  const uint32_t y = blockIdx.y, t = threadIdx.x;
  XYZZ<Fq> acc = XYZZ<Fq>::identity();
  for (size_t k = sg.lo[y] + blockIdx.x * (size_t)kSumThreads + t; k < sg.hi[y]; k += (size_t)gridDim.x * kSumThreads) xyzz_add(acc, T[k]);
  sh[t] = acc;
  __syncthreads();
  for (uint32_t w = kSumThreads / 2; w; w >>= 1) {
    if (t < w) xyzz_add(sh[t], sh[t + w]);
    __syncthreads();
  }
  if (t) return;
  if (out) out[y] = xyzz_to_affine(sh[0]);
  else partial[y * gridDim.x + blockIdx.x] = sh[0];
}

// one thread per pair of decoded points: its Miller value (1 when either point is the identity)
__global__ void __launch_bounds__(32) g16v_miller(const Affine<Fq>* P, const Affine<Fq2>* Q, size_t n, Fq12* f) {
  const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (k < n) f[k] = miller_pair(P[k], Q[k]);
}

// Tree product of Miller values, as g16v_sum: several CTAs write partial[blockIdx.x]; one CTA (the second launch) ends
// in the final exponentiation and writes *result = 1 when the product is one
__global__ void __launch_bounds__(kProdThreads) g16v_product(const Fq12* f, size_t n, Fq12* partial, uint8_t* result) {
  __shared__ Fq12 sh[kProdThreads];
  const uint32_t t = threadIdx.x;
  Fq12 acc = Fq12::one();
  for (size_t k = blockIdx.x * (size_t)kProdThreads + t; k < n; k += (size_t)gridDim.x * kProdThreads) acc = Fq12::mul(acc, f[k]);
  sh[t] = acc;
  __syncthreads();
  for (uint32_t w = kProdThreads / 2; w; w >>= 1) {
    if (t < w) sh[t] = Fq12::mul(sh[t], sh[t + w]);
    __syncthreads();
  }
  if (t) return;
  if (result) *result = Fq12::is_one(final_exponentiate(sh[0])) ? 1 : 0;
  else partial[blockIdx.x] = sh[0];
}

// The failure path, one thread per proof: its own check (-A_i, B_i) (alpha1, beta2) (vk_x(i), gamma2) (C_i, delta2) as
// pairs 4i .. 4i + 3, vk_x(i) = IC_0 + sum_j x_ij IC_j.  Every pair carries the proof's status, so pairing_check reports
// it; a malformed proof's pairs are identities.  Q holds B_0 .. B_n-1, then beta2, gamma2, delta2.
__global__ void __launch_bounds__(64) g16v_single(const uint8_t* x, uint32_t n_pub, const uint8_t* st, const Affine<Fq>* A, const Affine<Fq>* C,
                                                  const Affine<Fq2>* Q, const Affine<Fq>* g1, size_t n, Affine<Fq>* P4, Affine<Fq2>* Q4, uint8_t* pst4,
                                                  uint32_t* offs) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t s = st[i];
  Affine<Fq> p[4] = {g1_identity(), g1_identity(), g1_identity(), g1_identity()};
  if (!s) {
    XYZZ<Fq> vx = xyzz_from_affine(g1[1]);
    for (uint32_t j = 0; j < n_pub; ++j) {
      bool ok;
      const Fr xj = load_be<Fr>(x + 32 * (i * n_pub + j), &ok);
      xyzz_add(vx, xyzz_scalar_mul<Fq>(xj.v, g1[2 + j]));
    }
    p[0] = g1_neg(A[i]); p[1] = g1[0]; p[2] = xyzz_to_affine(vx); p[3] = C[i];
  }
  const Affine<Fq2> q[4] = {Q[i], Q[n], Q[n + 1], Q[n + 2]};
#pragma unroll
  for (int k = 0; k < 4; ++k) { P4[4 * i + k] = p[k]; Q4[4 * i + k] = q[k]; pst4[4 * i + k] = s; }
  offs[i] = (uint32_t)(4 * i);
  if (i + 1 == n) offs[n] = (uint32_t)(4 * n);
}

const char* const kVkNames[4] = {"alpha1", "beta2", "gamma2", "delta2"};

}  // namespace
}  // namespace b200zk

using namespace b200zk;

extern "C" int b200zk_groth16_verify_batch(b200zk_ctx* ctx, const uint8_t* vk, size_t vk_len, const uint8_t* proofs, const uint8_t* public_inputs,
                                           size_t count, uint8_t* valid, uint8_t* status, int* batch_ok) {
  static const char* what = "groth16_verify_batch";
  if (!ctx || !vk || (count && (!proofs || !valid || !status))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_verify_batch: null argument");
  NvtxRange nvtx("b200zk:groth16_verify_batch");
  DeviceGuard guard(ctx);
  if (vk_len < 512 || (vk_len - 448) % 64) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_verify_batch: vk_len must be 448 + 64 (n_pub + 1) bytes");
  const size_t n_ic = (vk_len - 448) / 64, n_pub = n_ic - 1, n = count;
  if (!n) return B200ZK_OK;
  if (n_pub && !public_inputs) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_verify_batch: null public_inputs");
  if (n > kMaxCount) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_verify_batch: more than 2^28 proofs in one call");
  if (n_ic > 65535) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_verify_batch: more than 65534 public inputs");
  cudaStream_t st = ctx->stream;
  uint8_t *d_proofs, *d_x, *d_vk, *d_rho, *d_st, *pst4, *res4, *sts4;
  Affine<Fq> *P, *A, *C, *g1, *P4;
  Affine<Fq2> *Q, *Q4;
  XYZZ<Fq> *T, *part;
  Fr* s;
  Fq12 *f, *fpart;
  uint32_t* offs;
  // d_st: the proofs' statuses, the vk elements' statuses and the combined check's result, read back in one copy
  const size_t n_out = n + 4 + n_ic + 1;
  B2_TRY(carve(ctx, ctx->ws_points, [&](Carve& c) {
    d_proofs = c.take<uint8_t>(256 * n); d_x = c.take<uint8_t>(32 * n * n_pub); d_vk = c.take<uint8_t>(vk_len); d_rho = c.take<uint8_t>(16 * n);
    P = c.take<Affine<Fq>>(n + 3); Q = c.take<Affine<Fq2>>(n + 3); A = c.take<Affine<Fq>>(n); C = c.take<Affine<Fq>>(n); g1 = c.take<Affine<Fq>>(1 + n_ic);
    T = c.take<XYZZ<Fq>>(n + n_ic); s = c.take<Fr>(n_ic); part = c.take<XYZZ<Fq>>(2 * kSumBlocks); f = c.take<Fq12>(4 * n + 3); fpart = c.take<Fq12>(kProdBlocks);
    d_st = c.take<uint8_t>(n_out);
    P4 = c.take<Affine<Fq>>(4 * n); Q4 = c.take<Affine<Fq2>>(4 * n); pst4 = c.take<uint8_t>(4 * n); offs = c.take<uint32_t>(n + 1);
    res4 = c.take<uint8_t>(n); sts4 = c.take<uint8_t>(n);
  }));
  uint8_t* vst = d_st + n;
  uint8_t* d_ok = d_st + n + 4 + n_ic;
  // 1. decode and validate the key and the proofs; the host hashes meanwhile
  B2_CUDA(ctx, cudaMemcpyAsync(d_proofs, proofs, 256 * n, cudaMemcpyHostToDevice, st));
  if (n_pub) B2_CUDA(ctx, cudaMemcpyAsync(d_x, public_inputs, 32 * n * n_pub, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(d_vk, vk, vk_len, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, g16v_vk_decode, (unsigned)((4 + n_ic + 63) / 64), 64, 0, st, (const uint8_t*)d_vk, (uint32_t)n_ic, g1, Q + n, vst);
  B2_LAUNCH(ctx, g16v_decode, (unsigned)((n + 63) / 64), 64, 0, st, (const uint8_t*)d_proofs, (const uint8_t*)d_x, (uint32_t)n_pub, n, A, Q, C, d_st);
  // 2. rho_i = the first 16 bytes, big-endian, of SHA-256(D | i as u64 BE), 1 if those are all zero, where
  //    D = SHA-256("b200zk-groth16-batch-v1" | vk | count as u64 BE | proofs | public inputs)
  static const char kTag[] = "b200zk-groth16-batch-v1";
  uint8_t be[8], digest[32];
  auto put_u64 = [&](uint64_t v) { for (int k = 0; k < 8; ++k) be[7 - k] = (uint8_t)(v >> (8 * k)); };
  Sha256 h;
  h.update((const uint8_t*)kTag, sizeof kTag - 1);
  h.update(vk, vk_len);
  put_u64(n);
  h.update(be, 8);
  h.update(proofs, 256 * n);
  if (n_pub) h.update(public_inputs, 32 * n * n_pub);
  h.final(digest);
  std::vector<uint8_t> h_rho(16 * n);
  for (size_t i = 0; i < n; ++i) {
    Sha256 hi;
    hi.update(digest, 32);
    put_u64(i);
    hi.update(be, 8);
    uint8_t d[32];
    hi.final(d);
    uint8_t any = 0;
    for (int k = 0; k < 16; ++k) any |= d[k];
    if (!any) d[15] = 1;
    memcpy(&h_rho[16 * i], d, 16);
  }
  B2_CUDA(ctx, cudaMemcpyAsync(d_rho, h_rho.data(), 16 * n, cudaMemcpyHostToDevice, st));
  // 3. the combined check's pairs: P[i] = -rho_i A_i with Q[i] = B_i; P[n] = s_0 alpha1, P[n + 1] = sum_j s_j IC_j,
  //    P[n + 2] = sum_i rho_i C_i with Q[n ..] = beta2, gamma2, delta2
  B2_LAUNCH(ctx, g16v_terms, (unsigned)((n + 63) / 64), 64, 0, st, (const uint8_t*)d_rho, (const uint8_t*)d_st, (const Affine<Fq>*)A, (const Affine<Fq>*)C, n, P, T);
  B2_LAUNCH(ctx, g16v_scalars, (unsigned)n_ic, kScalarThreads, 0, st, (const uint8_t*)d_rho, (const uint8_t*)d_st, (const uint8_t*)d_x, (uint32_t)n_pub, n, s);
  B2_LAUNCH(ctx, g16v_vk_terms, (unsigned)((n_ic + 1 + 63) / 64), 64, 0, st, (const Fr*)s, (const Affine<Fq>*)g1, (uint32_t)n_ic, T + n, P + n);
  const Segs sg = {{n, 0}, {n + n_ic, n}};  // segment 0: the IC terms -> P[n + 1]; segment 1: the rho_i C_i -> P[n + 2]
  const unsigned sum_blocks = (unsigned)std::min<size_t>(kSumBlocks, (n + kSumThreads - 1) / kSumThreads);
  const Segs sg2 = {{0, sum_blocks}, {sum_blocks, 2 * (size_t)sum_blocks}};
  B2_LAUNCH(ctx, g16v_sum, dim3(sum_blocks, 2), kSumThreads, 0, st, (const XYZZ<Fq>*)T, sg, part, (Affine<Fq>*)nullptr);
  B2_LAUNCH(ctx, g16v_sum, dim3(1, 2), kSumThreads, 0, st, (const XYZZ<Fq>*)part, sg2, (XYZZ<Fq>*)nullptr, P + n + 1);
  // 4. N + 3 Miller loops, a tree product, one final exponentiation
  const unsigned prod_blocks = (unsigned)std::min<size_t>(kProdBlocks, (n + 3 + kProdThreads - 1) / kProdThreads);
  B2_LAUNCH(ctx, g16v_miller, (unsigned)((n + 3 + 31) / 32), 32, 0, st, (const Affine<Fq>*)P, (const Affine<Fq2>*)Q, n + 3, f);
  B2_LAUNCH(ctx, g16v_product, prod_blocks, kProdThreads, 0, st, (const Fq12*)f, n + 3, fpart, (uint8_t*)nullptr);
  B2_LAUNCH(ctx, g16v_product, 1, kProdThreads, 0, st, (const Fq12*)fpart, (size_t)prod_blocks, (Fq12*)nullptr, d_ok);
  std::vector<uint8_t> h_out(n_out);
  B2_CUDA(ctx, cudaMemcpyAsync(h_out.data(), d_st, n_out, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  // a refused key fails the call (a coordinate >= p anywhere in it outranks a curve error), naming the element
  for (const uint8_t want : {(uint8_t)B200ZK_ERR_NOT_IN_FIELD, (uint8_t)B200ZK_ERR_NOT_ON_CURVE}) {
    for (size_t e = 0; e < 4 + n_ic; ++e) {
      if (h_out[n + e] != want) continue;
      char name[32], msg[160];
      if (e < 4) snprintf(name, sizeof name, "%s", kVkNames[e]);
      else snprintf(name, sizeof name, "IC[%zu]", e - 4);
      snprintf(msg, sizeof msg, "%s: vk %s %s", what, name,
               want == B200ZK_ERR_NOT_IN_FIELD ? "has a coordinate >= p" : (e >= 1 && e < 4 ? "is not on the twist or not in the order-r subgroup" : "is not on the curve"));
      return fail(ctx, want, msg);
    }
  }
  if (h_out[n_out - 1]) {
    for (size_t i = 0; i < n; ++i) { valid[i] = h_out[i] ? 0 : 1; status[i] = h_out[i]; }
    if (batch_ok) *batch_ok = 1;
    return B200ZK_OK;
  }
  // 5. the combined check failed: every proof's own 4-pair check
  B2_LAUNCH(ctx, g16v_single, (unsigned)((n + 63) / 64), 64, 0, st, (const uint8_t*)d_x, (uint32_t)n_pub, (const uint8_t*)d_st, (const Affine<Fq>*)A,
            (const Affine<Fq>*)C, (const Affine<Fq2>*)Q, (const Affine<Fq>*)g1, n, P4, Q4, pst4, offs);
  B2_LAUNCH(ctx, g16v_miller, (unsigned)((4 * n + 31) / 32), 32, 0, st, (const Affine<Fq>*)P4, (const Affine<Fq2>*)Q4, 4 * n, f);
  B2_LAUNCH(ctx, (pairing_check<Fq12, final_exponentiate>), (unsigned)((n + 31) / 32), 32, 0, st, (const Fq12*)f, (const uint8_t*)pst4, (const uint32_t*)offs, n, res4, sts4);
  std::vector<uint8_t> h_res(n);
  B2_CUDA(ctx, cudaMemcpyAsync(h_res.data(), res4, n, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  for (size_t i = 0; i < n; ++i) { valid[i] = (h_res[i] && !h_out[i]) ? 1 : 0; status[i] = h_out[i]; }
  if (batch_ok) *batch_ok = 0;
  return B200ZK_OK;
}
