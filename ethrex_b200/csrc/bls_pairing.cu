// bls_pairing.cu -- the BLS12-381 pairing on the device and the three calls of the reference that rest on it:
//   the EIP-2537 pairing check        Crypto::bls12_381_pairing_check, /root/reference/crates/common/crypto/provider.rs:642-672
//   verify_kzg_proof (0x0a precompile) Crypto::verify_kzg_proof, provider.rs:463-507 (levm precompiles.rs:923-985)
//   verify_blob_kzg_proof_batch        BlobsBundle::verify_kzg_proofs -> kzg::verify_kzg_proof_batch (blobs_bundle.rs:155-173,
//                                      kzg.rs:168-192); verify_blob_kzg_proof (provider.rs:509-544) is its batch of one
//
// Tower: Fp2 = Fp[u]/(u^2 + 1) (bls12.cuh), Fp6 = Fp2[v]/(v^3 - (1 + u)), Fp12 = Fp6[w]/(w^2 - v) (tower.cuh).  The
// twist is M-type: E': y^2 = x^3 + 4(1 + u).
// Miller loop: optimal ate over |x| = 0xd201000000010000 (64 bits: 63 doublings, 5 additions).  The line coefficients of a
// G2 point depend on that point only, so a prepare pass (one thread per G2 point) writes its 68 triples in homogeneous
// projective coordinates -- no inversion anywhere -- and the Miller kernel (one thread per pair) only evaluates them at P:
// the G2Prepared + multi_miller_loop split of provider.rs:651-670.  x is negative: f is conjugated at the end.
// Final exponentiation: the easy part f^((p^6 - 1)(p^2 + 1)) (conjugate, one inversion, one p^2 Frobenius), then the hard
// part through the x-chain 3 (p^4 - p^2 + 1)/r = (x - 1)^2 (x + p) (x^2 + p^2 - 1) + 3: five exponentiations by x, three
// Frobenius maps and a handful of products instead of a generic 1269-bit power.  It yields the CUBE of the reduced pairing;
// a check asks whether a product of pairings is one, and since gcd(3, r) = 1, z^3 = 1 exactly when z = 1 for z in the
// order-r group mu_r.  tests/test_bls12_pairing_host.py recomputes every constant of this file and of
// bls_pairing.cuh, which holds the pairing's stages, and checks the identity.
#include "bls_pairing.cuh"
#include "cell_batch.h"
#include "sha256.h"
#include <cstring>
#include <vector>

namespace b200zk {
namespace {

// the G1 generator (x, y), canonical limbs
__constant__ uint32_t kG1Gen[2][12] = {
    {0xdb22c6bbu, 0xfb3af00au, 0xf97a1aefu, 0x6c55e83fu, 0x171bac58u, 0xa14e3a3fu, 0x9774b905u, 0xc3688c4fu, 0x4fa9ac0fu, 0x2695638cu, 0x3197d794u, 0x17f1d3a7u},
    {0x46c5e7e1u, 0x0caa2329u, 0xa2888ae4u, 0xd03cc744u, 0x2c04b3edu, 0x00db18cbu, 0xd5d00af6u, 0xfcf5e095u, 0x741d8ae4u, 0xa09e30edu, 0xe3aaa0f1u, 0x08b3f481u}};
// the G2 generator in the 96-byte compressed form (a published constant): point 0 of a KZG G2 setup must be this
const uint8_t kG2GenCompressed[96] = {
    0x93, 0xe0, 0x2b, 0x60, 0x52, 0x71, 0x9f, 0x60, 0x7d, 0xac, 0xd3, 0xa0, 0x88, 0x27, 0x4f, 0x65, 0x59, 0x6b, 0xd0, 0xd0, 0x99, 0x20, 0xb6, 0x1a,
    0xb5, 0xda, 0x61, 0xbb, 0xdc, 0x7f, 0x50, 0x49, 0x33, 0x4c, 0xf1, 0x12, 0x13, 0x94, 0x5d, 0x57, 0xe5, 0xac, 0x7d, 0x05, 0x5d, 0x04, 0x2b, 0x7e,
    0x02, 0x4a, 0xa2, 0xb2, 0xf0, 0x8f, 0x0a, 0x91, 0x26, 0x08, 0x05, 0x27, 0x2d, 0xc5, 0x10, 0x51, 0xc6, 0xe4, 0x7a, 0xd4, 0xfa, 0x40, 0x3b, 0x02,
    0xb4, 0x51, 0x0b, 0x64, 0x7a, 0xe3, 0xd1, 0x77, 0x0b, 0xac, 0x03, 0x26, 0xa8, 0x05, 0xbb, 0xef, 0xd4, 0x80, 0x56, 0xc8, 0xc1, 0x21, 0xbd, 0xb8};

// ---- kernels ----------------------------------------------------------------------------------------------------------
// one thread per (G1, G2) pair of EIP-2537 bytes (128 + 256): range and padding (status 2), then curve and subgroup of
// both points (status 3); kTrivial when a side is the identity
__global__ void __launch_bounds__(64) bls_pair_decode(const uint8_t* __restrict__ pairs, size_t n, Affine<Fp381>* P, Affine<F2>* Q, uint8_t* pst) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* src = pairs + 384 * i;
  Fp381 c[6];
  bool in_range = true;
#pragma unroll 1
  for (int k = 0; k < 6; ++k) in_range &= load_fp64(src + 64 * k, &c[k]);
  Affine<Fp381> p = {Fp381::zero(), Fp381::zero()};
  Affine<F2> q = {F2::zero(), F2::zero()};
  uint32_t s = 0;
  if (!in_range) s = B200ZK_ERR_NOT_IN_FIELD;
  else {
    p = {Fp381::to_mont(c[0]), Fp381::to_mont(c[1])};
    q = {{Fp381::to_mont(c[2]), Fp381::to_mont(c[3])}, {Fp381::to_mont(c[4]), Fp381::to_mont(c[5])}};
    if (!affine_on_curve(p) || !affine_on_curve(q)) s = B200ZK_ERR_NOT_ON_CURVE;
    else if ((!p.is_inf() && !in_subgroup<bls_r_limb>(p)) || (!q.is_inf() && !in_subgroup<bls_r_limb>(q))) s = B200ZK_ERR_NOT_ON_CURVE;
  }
  if (!s && (p.is_inf() || q.is_inf())) s = kTrivial;
  P[i] = p;
  Q[i] = q;
  pst[i] = (uint8_t)s;
}

// 96-byte compressed G2 points (x.c1 | x.c0, flags in byte 0) -> native affine, subgroup-checked.  status[0] / [1]: first
// index with a coordinate >= p / with bad flags, off the curve or outside the subgroup (atomicMin; initialised to n)
__global__ void __launch_bounds__(64) bls_g2_decode(const uint8_t* __restrict__ in, size_t n, Affine<F2>* out, unsigned long long* status) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* src = in + 96 * i;
  const uint8_t flags = src[0];
  const bool c_flag = flags & 0x80, inf_flag = flags & 0x40, sign_flag = flags & 0x20;
  const Fp381 x1 = load_be48(src, 0x1fffffffu), x0 = load_be48(src + 48, 0xffffffffu);
  Affine<F2> pt = {F2::zero(), F2::zero()};
  bool bad_field = false, bad_point = false;
  if (!c_flag) bad_point = true;
  else if (inf_flag) { if (sign_flag || !x0.is_zero() || !x1.is_zero()) bad_point = true; }
  else if (!Fp381::less(x0, Fp381::modulus()) || !Fp381::less(x1, Fp381::modulus())) bad_field = true;
  else {
    const F2 x = {Fp381::to_mont(x0), Fp381::to_mont(x1)};
    const F2 rhs = F2::add(F2::mul(F2::sqr(x), x), CurveB<F2>::b());
    F2 y = F2::sqrt_candidate(rhs);
    if (F2::sqr(y) != rhs) bad_point = true;
    else {
      const Fp381 half = fp381_half(), y0 = Fp381::from_mont(y.c0), y1 = Fp381::from_mont(y.c1);
      const bool larger = Fp381::less(half, y1) || (y1.is_zero() && Fp381::less(half, y0));
      if (larger != sign_flag) y = F2::neg(y);
      pt = {x, y};
      if (!in_subgroup<bls_r_limb>(pt)) bad_point = true;
    }
  }
  if (bad_field) atomicMin(status, (unsigned long long)i);
  if (bad_point) atomicMin(status + 1, (unsigned long long)i);
  if (bad_field || bad_point) pt = {F2::zero(), F2::zero()};
  out[i] = pt;
}

// one thread per G2 point: its 68 line triples (skipped where pst marks the pair bad or trivial, or Q is the identity)
__global__ void __launch_bounds__(64) bls_g2_prepare(const Affine<F2>* Q, const uint8_t* pst, size_t n, BlsLine* lines) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n || (pst && pst[i])) return;
  const Affine<F2> q = Q[i];
  if (!q.is_inf()) g2_prepare(q, lines + kLines * i);
}

// one thread per pair: the Miller value over prepared lines (pair i uses line set i, or i % period when period != 0)
__global__ void __launch_bounds__(32) bls_miller(const Affine<Fp381>* P, const BlsLine* lines, uint32_t period, const uint8_t* pst, size_t n, F12* f) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  F12 r = F12::one();
  if (!pst[i]) r = miller_prepared(lines + kLines * (period ? i % period : i), P[i]);
  f[i] = r;
}

// c-kzg validate_kzg_g1 on 48-byte compressed points: decompression (status 2 / 3) and r P = O (status 3); identity valid
__global__ void __launch_bounds__(64) bls_g1_decode_subgroup(const uint8_t* __restrict__ in, size_t n, Affine<Fp381>* out, uint8_t* st) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<Fp381> p;
  uint32_t s = bls_g1_decompress(in + 48 * i, &p);
  if (!s && !p.is_inf() && !in_subgroup<bls_r_limb>(p)) s = B200ZK_ERR_NOT_ON_CURVE;
  if (s) p = {Fp381::zero(), Fp381::zero()};
  out[i] = p;
  st[i] = (uint8_t)s;
}

B2_D Affine<Fp381> g1_generator() { return {fp_const(kG1Gen[0]), fp_const(kG1Gen[1])}; }
B2_D Affine<Fp381> affine_neg(const Affine<Fp381>& p) { return {p.x, Fp381::neg(p.y)}; }

// verify_kzg_proof per item: e(C - [y]G1, G2) = e(pi, [tau - z]G2) is rewritten as e(C - [y]G1 + [z]pi, G2) e(-pi, [tau]G2) = 1,
// so both G2 points are fixed.  pts = n commitments, then n proofs (decoded, with their statuses).  Out: pair 2i = the first
// G1 point, pair 2i + 1 = -pi, both with the item's status
__global__ void __launch_bounds__(64) kzg_verify_combine(const Affine<Fp381>* pts, const uint8_t* pt_st, const uint8_t* __restrict__ z_be,
                                                          const uint8_t* __restrict__ y_be, size_t n, Affine<Fp381>* P, uint8_t* pst) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const Fr381 z = load_be32(z_be + 32 * i), y = load_be32(y_be + 32 * i);
  const uint32_t sc = pt_st[i], sp = pt_st[n + i];
  uint32_t s = 0;
  if (!Fr381::less(z, Fr381::modulus()) || !Fr381::less(y, Fr381::modulus()) || sc == B200ZK_ERR_NOT_IN_FIELD || sp == B200ZK_ERR_NOT_IN_FIELD) s = B200ZK_ERR_NOT_IN_FIELD;
  else if (sc || sp) s = B200ZK_ERR_NOT_ON_CURVE;
  Affine<Fp381> p1 = {Fp381::zero(), Fp381::zero()}, p2 = p1;
  if (!s) {
    const Affine<Fp381> c = pts[i], pi = pts[n + i];
    XYZZ<Fp381> acc = xyzz_scalar_mul<Fp381>(z.v, pi);
    xyzz_add_mixed(acc, c.x, c.y);
    XYZZ<Fp381> yg = xyzz_scalar_mul<Fp381>(y.v, g1_generator());
    yg.y = Fp381::neg(yg.y);
    xyzz_add(acc, yg);
    p1 = xyzz_to_affine(acc);
    p2 = affine_neg(pi);
  }
  P[2 * i] = p1;
  P[2 * i + 1] = p2;
  pst[2 * i] = (uint8_t)(s ? s : (p1.is_inf() ? kTrivial : 0));
  pst[2 * i + 1] = (uint8_t)(s ? s : (p2.is_inf() ? kTrivial : 0));
}

// verify_blob_kzg_proof_batch, one thread per blob: with rho = the batch's random challenge,
//   terms[i] = [rho^i] C_i - [rho^i y_i] G1 + [rho^i z_i] pi_i,   terms[n + i] = [rho^i] pi_i
__global__ void __launch_bounds__(64) kzg_blob_terms(const Affine<Fp381>* pts, const uint8_t* __restrict__ z_be, const uint8_t* __restrict__ y_be,
                                                      const uint8_t* __restrict__ rho_be, size_t n, XYZZ<Fp381>* terms) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint32_t e[8] = {(uint32_t)i, (uint32_t)((uint64_t)i >> 32), 0, 0, 0, 0, 0, 0};
  const Fr381 ri = Fr381::pow(Fr381::to_mont(load_be32(rho_be)), e);  // Montgomery
  // mul(canonical, Montgomery) is the canonical product
  const Fr381 ri_c = Fr381::from_mont(ri), rz = Fr381::mul(load_be32(z_be + 32 * i), ri), ry = Fr381::mul(load_be32(y_be + 32 * i), ri);
  const Affine<Fp381> c = pts[i], pi = pts[n + i];
  XYZZ<Fp381> b = xyzz_scalar_mul<Fp381>(ri_c.v, c);
  xyzz_add(b, xyzz_scalar_mul<Fp381>(rz.v, pi));
  XYZZ<Fp381> yg = xyzz_scalar_mul<Fp381>(ry.v, g1_generator());
  yg.y = Fp381::neg(yg.y);
  xyzz_add(b, yg);
  terms[i] = b;
  terms[n + i] = xyzz_scalar_mul<Fp381>(ri_c.v, pi);
}

// one thread: P[0] = sum of terms[0..n), P[1] = -(sum of terms[n..2n)) -- the batch's single 2-pair check
__global__ void __launch_bounds__(32) kzg_blob_fold(const XYZZ<Fp381>* terms, size_t n, Affine<Fp381>* P, uint8_t* pst) {
  if (blockIdx.x || threadIdx.x) return;
  XYZZ<Fp381> b = XYZZ<Fp381>::identity(), a = XYZZ<Fp381>::identity();
#pragma unroll 1
  for (size_t k = 0; k < n; ++k) { xyzz_add(b, terms[k]); xyzz_add(a, terms[n + k]); }
  const Affine<Fp381> p1 = xyzz_to_affine(b), p2 = affine_neg(xyzz_to_affine(a));
  P[0] = p1;
  P[1] = p2;
  pst[0] = p1.is_inf() ? kTrivial : 0;
  pst[1] = p2.is_inf() ? kTrivial : 0;
}

// verify_cell_kzg_proof_batch from its three MSMs (parts: sum r^k pi_k | the commitments' and r^k h_k^64 pi_k terms |
// [sum r^k I_k(tau)]1): P[0] = parts[1] - parts[2], paired with G2; P[1] = -parts[0], paired with [tau^64]2
__global__ void __launch_bounds__(32) kzg_cell_fold(const XYZZ<Fp381>* parts, Affine<Fp381>* P, uint8_t* pst) {
  if (blockIdx.x || threadIdx.x) return;
  XYZZ<Fp381> b = parts[1], i = parts[2];
  i.y = Fp381::neg(i.y);
  xyzz_add(b, i);
  const Affine<Fp381> p1 = xyzz_to_affine(b), p2 = affine_neg(xyzz_to_affine(parts[0]));
  P[0] = p1;
  P[1] = p2;
  pst[0] = p1.is_inf() ? kTrivial : 0;
  pst[1] = p2.is_inf() ? kTrivial : 0;
}

// ---- host side ----------------------------------------------------------------------------------------------------------
size_t g2_lines_offset(size_t n) { return (n * sizeof(Affine<F2>) + 255) & ~(size_t)255; }
const BlsLine* g2_setup_lines(const BasesEntry& e) { return reinterpret_cast<const BlsLine*>((const uint8_t*)e.d.p + g2_lines_offset(e.n)); }

// the G2 handle of a KZG verification: BLS12-381 G2, at least 2 points, point 0 the generator (point 1 is then [tau]2)
int kzg_g2_setup(b200zk_ctx* ctx, uint64_t handle, const char* what, const BasesEntry** e) {
  std::string msg = what;
  *e = find_bases(ctx, handle, Group::Bls12G2, (msg + ": unknown BLS12-381 G2 setup handle").c_str());
  if (!*e) return B200ZK_ERR_INVALID_ARG;
  if ((*e)->n < 2) return fail(ctx, B200ZK_ERR_INVALID_ARG, (msg + ": the G2 setup must hold at least 2 points").c_str());
  if (!(*e)->g2_gen0) return fail(ctx, B200ZK_ERR_INVALID_ARG, (msg + ": point 0 of the G2 setup is not the G2 generator").c_str());
  return B200ZK_OK;
}

// Miller values of n_pairs pairs (line set i, or i % period), then `count` checks over d_offsets
int pairing_run(b200zk_ctx* ctx, const Affine<Fp381>* P, const BlsLine* lines, uint32_t period, const uint8_t* pst, size_t n_pairs,
                const uint32_t* offsets, size_t count, F12* f, uint8_t* result, uint8_t* status, cudaStream_t st) {
  if (n_pairs) B2_LAUNCH(ctx, bls_miller, (unsigned)((n_pairs + 31) / 32), 32, 0, st, P, lines, period, pst, n_pairs, f);
  B2_LAUNCH(ctx, (pairing_check<F12, final_exponentiate>), (unsigned)((count + 31) / 32), 32, 0, st, (const F12*)f, pst, offsets, count, result, status);
  return B200ZK_OK;
}

// the handles of a cell-proof check: the 4096-point Lagrange G1 setup, and a G2 setup of at least 65 points whose point 0
// is the generator (point 64 is [tau^64]2)
int cell_setups(b200zk_ctx* ctx, uint64_t g1_setup, uint64_t g2_setup, const char* what, const BasesEntry** g1, const BasesEntry** g2) {
  const std::string msg = what;
  *g1 = find_bases(ctx, g1_setup, Group::Bls12G1, (msg + ": unknown G1 setup handle").c_str());
  if (!*g1) return B200ZK_ERR_INVALID_ARG;
  if ((*g1)->n != 4096) return fail(ctx, B200ZK_ERR_INVALID_ARG, (msg + ": the G1 setup must hold FIELD_ELEMENTS_PER_BLOB = 4096 points").c_str());
  B2_TRY(kzg_g2_setup(ctx, g2_setup, what, g2));
  if ((*g2)->n < 65) return fail(ctx, B200ZK_ERR_INVALID_ARG, (msg + ": the G2 setup must hold at least 65 points ([tau^64]2 is point 64)").c_str());
  return B200ZK_OK;
}

// the workspace of cell_check_tail, carved behind the caller's own buffers
struct CellTail {
  XYZZ<Fp381>* parts;
  Affine<F2>* q2;
  BlsLine* lines;
  Affine<Fp381>* P;
  uint8_t* pst;
  F12* f;
  uint32_t* offs;
  uint8_t* res;
  uint8_t* sts;
  void take(Carve& c) {
    parts = c.take<XYZZ<Fp381>>(3); q2 = c.take<Affine<F2>>(2); lines = c.take<BlsLine>(2 * kLines);
    P = c.take<Affine<Fp381>>(2); pst = c.take<uint8_t>(2); f = c.take<F12>(2); offs = c.take<uint32_t>(2); res = c.take<uint8_t>(1); sts = c.take<uint8_t>(1);
  }
};

// The end of both cell-proof checks, from their scalars on the device: three MSMs (sum r^k pi_k over the m proofs; the
// n_c commitments' weights and the r^k h_k^64 pi_k terms over pts = the n_c commitments then the m proofs; [A(tau)]1 over
// the Lagrange setup with its window table), kzg_cell_fold, and one 2-pair check against (G2, [tau^64]2) into *valid
int cell_check_tail(b200zk_ctx* ctx, const BasesEntry& g1, const BasesEntry& g2, const Affine<Fp381>* pts, size_t n_c, size_t m, const void* s_proof,
                    const void* s_lin, const void* s_setup, const CellTail& w, cudaStream_t st, int* valid) {
  B2_TRY(msm_run_bls(ctx, pts + n_c, s_proof, m, 0, st, w.parts));
  B2_TRY(msm_run_bls(ctx, pts, s_lin, n_c + m, 0, st, w.parts + 1));
  B2_TRY(msm_run_bls(ctx, g1.d.p, s_setup, g1.n, 0, st, w.parts + 2, g1.table_c, g1.n));
  B2_LAUNCH(ctx, kzg_cell_fold, 1, 32, 0, st, (const XYZZ<Fp381>*)w.parts, w.P, w.pst);
  const Affine<F2>* g2pts = (const Affine<F2>*)g2.d.p;
  B2_CUDA(ctx, cudaMemcpyAsync(w.q2, g2pts, sizeof(Affine<F2>), cudaMemcpyDeviceToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(w.q2 + 1, g2pts + 64, sizeof(Affine<F2>), cudaMemcpyDeviceToDevice, st));
  B2_LAUNCH(ctx, bls_g2_prepare, 1, 64, 0, st, (const Affine<F2>*)w.q2, (const uint8_t*)nullptr, (size_t)2, w.lines);
  const uint32_t h_offs[2] = {0, 2};
  B2_CUDA(ctx, cudaMemcpyAsync(w.offs, h_offs, 8, cudaMemcpyHostToDevice, st));
  B2_TRY(pairing_run(ctx, w.P, w.lines, 2, w.pst, 2, w.offs, 1, w.f, w.res, w.sts, st));
  uint8_t h_res = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(&h_res, w.res, 1, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  *valid = h_res ? 1 : 0;
  return B200ZK_OK;
}

}  // namespace
}  // namespace b200zk

using namespace b200zk;

extern "C" {

int b200zk_bls12_381_g2_bases_upload(b200zk_ctx* ctx, const void* points, size_t n, uint32_t flags, uint64_t* handle) {
  if (!ctx || !handle || (!points && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bls12_381_g2_bases_upload: null argument");
  if (!(flags & B200ZK_POINTS_COMPRESSED)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bls12_381_g2_bases_upload: points must be 96-byte compressed (B200ZK_POINTS_COMPRESSED)");
  DeviceGuard guard(ctx);
  cudaStream_t st = ctx->stream;
  BasesEntry e;
  e.n = n; e.group = Group::Bls12G2;
  const size_t lines_off = g2_lines_offset(n);
  B2_TRY(ensure(ctx, ctx->ws_pairing, n * 96 + 256 + 16));
  B2_CUDA(ctx, cudaMalloc(&e.d.p, lines_off + 2 * kLines * sizeof(BlsLine) + 32));
  unsigned long long* d_status = (unsigned long long*)((uint8_t*)ctx->ws_pairing.p + ((n * 96 + 255) & ~(size_t)255));
  unsigned long long h[2] = {(unsigned long long)n, (unsigned long long)n};
  int rc = B200ZK_OK;
  cudaError_t ce = cudaMemcpyAsync(d_status, h, 16, cudaMemcpyHostToDevice, st);
  if (ce == cudaSuccess && n) ce = cudaMemcpyAsync(ctx->ws_pairing.p, points, n * 96, cudaMemcpyHostToDevice, st);
  if (ce == cudaSuccess && n) {
    bls_g2_decode<<<(unsigned)((n + 63) / 64), 64, 0, st>>>((const uint8_t*)ctx->ws_pairing.p, n, (Affine<F2>*)e.d.p, d_status);
    ctx->launches++;
    ce = cudaGetLastError();
  }
  if (ce == cudaSuccess) ce = cudaMemcpyAsync(h, d_status, 16, cudaMemcpyDeviceToHost, st);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
  if (ce == cudaSuccess && h[0] < n && h[0] <= h[1]) rc = fail(ctx, B200ZK_ERR_NOT_IN_FIELD, "bls12-381 G2 point: coordinate >= p");
  else if (ce == cudaSuccess && h[1] < n) rc = fail(ctx, B200ZK_ERR_NOT_ON_CURVE, "bls12-381 G2 point: malformed flag bits, not on the twist or not in the order-r subgroup");
  // the lines of points 0 and 1 (G2 and [tau]2 of a KZG setup), once per handle: the upload is synchronous, so they are
  // ready before the handle is returned
  if (ce == cudaSuccess && rc == B200ZK_OK && n >= 2) {
    bls_g2_prepare<<<1, 64, 0, st>>>((const Affine<F2>*)e.d.p, nullptr, 2, (BlsLine*)((uint8_t*)e.d.p + lines_off));
    ctx->launches++;
    ce = cudaGetLastError();
    if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
  }
  if (rc != B200ZK_OK) return rc;
  if (ce != cudaSuccess) return fail(ctx, B200ZK_ERR_CUDA, "bls12_381_g2_bases_upload", ce);
  e.g2_gen0 = n >= 1 && memcmp(points, kG2GenCompressed, 96) == 0;  // a valid point has one encoding
  return register_bases(ctx, std::move(e), handle);
}

int b200zk_bls12_381_pairing_check_batch(b200zk_ctx* ctx, const uint8_t* pairs, const uint32_t* pair_offsets, size_t count, uint8_t* result, uint8_t* status) {
  if (!ctx || (count && (!pair_offsets || !result || !status))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bls12_381_pairing_check_batch: null argument");
  if (count && pair_offsets[count] && !pairs) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bls12_381_pairing_check_batch: null pairs");
  NvtxRange nvtx("b200zk:bls12_381_pairing_check_batch");
  DeviceGuard guard(ctx);
  if (!count) return B200ZK_OK;
  B2_TRY(check_offsets(ctx, pair_offsets, count, "bls12_381_pairing_check_batch"));
  const size_t n = pair_offsets[count];
  cudaStream_t st = ctx->stream;
  uint8_t *in, *pst, *res, *sts;
  Affine<Fp381>* P;
  Affine<F2>* Q;
  BlsLine* lines;
  F12* f;
  uint32_t* offs;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    in = c.take<uint8_t>(384 * n); P = c.take<Affine<Fp381>>(n); Q = c.take<Affine<F2>>(n); pst = c.take<uint8_t>(n);
    lines = c.take<BlsLine>(kLines * n); f = c.take<F12>(n); offs = c.take<uint32_t>(count + 1); res = c.take<uint8_t>(count); sts = c.take<uint8_t>(count);
  }));
  if (n) B2_CUDA(ctx, cudaMemcpyAsync(in, pairs, 384 * n, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(offs, pair_offsets, (count + 1) * 4, cudaMemcpyHostToDevice, st));
  if (n) {
    B2_LAUNCH(ctx, bls_pair_decode, (unsigned)((n + 63) / 64), 64, 0, st, (const uint8_t*)in, n, P, Q, pst);
    B2_LAUNCH(ctx, bls_g2_prepare, (unsigned)((n + 63) / 64), 64, 0, st, (const Affine<F2>*)Q, (const uint8_t*)pst, n, lines);
  }
  B2_TRY(pairing_run(ctx, P, lines, 0, pst, n, offs, count, f, res, sts, st));
  B2_CUDA(ctx, cudaMemcpyAsync(result, res, count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(status, sts, count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

int b200zk_kzg_verify_proof_batch(b200zk_ctx* ctx, uint64_t g2_setup, const uint8_t* commitments, const uint8_t* z, const uint8_t* y,
                                  const uint8_t* proofs, size_t n, uint8_t* result, uint8_t* status) {
  static const char* what = "kzg_verify_proof_batch";
  if (!ctx || (n && (!commitments || !z || !y || !proofs || !result || !status))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_verify_proof_batch: null argument");
  NvtxRange nvtx("b200zk:kzg_verify_proof_batch");
  DeviceGuard guard(ctx);
  const BasesEntry* e = nullptr;
  B2_TRY(kzg_g2_setup(ctx, g2_setup, what, &e));
  if (!n) return B200ZK_OK;
  cudaStream_t st = ctx->stream;
  uint8_t *in, *zb, *yb, *pt_st, *pst, *res, *sts;
  Affine<Fp381>*pts, *P;
  F12* f;
  uint32_t* offs;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    in = c.take<uint8_t>(96 * n); zb = c.take<uint8_t>(32 * n); yb = c.take<uint8_t>(32 * n); pts = c.take<Affine<Fp381>>(2 * n);
    pt_st = c.take<uint8_t>(2 * n); P = c.take<Affine<Fp381>>(2 * n); pst = c.take<uint8_t>(2 * n); f = c.take<F12>(2 * n);
    offs = c.take<uint32_t>(n + 1); res = c.take<uint8_t>(n); sts = c.take<uint8_t>(n);
  }));
  std::vector<uint32_t> h_offs(n + 1);
  for (size_t i = 0; i <= n; ++i) h_offs[i] = (uint32_t)(2 * i);
  B2_CUDA(ctx, cudaMemcpyAsync(in, commitments, 48 * n, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(in + 48 * n, proofs, 48 * n, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(zb, z, 32 * n, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(yb, y, 32 * n, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(offs, h_offs.data(), 4 * (n + 1), cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, bls_g1_decode_subgroup, (unsigned)((2 * n + 63) / 64), 64, 0, st, (const uint8_t*)in, 2 * n, pts, pt_st);
  B2_LAUNCH(ctx, kzg_verify_combine, (unsigned)((n + 63) / 64), 64, 0, st, (const Affine<Fp381>*)pts, (const uint8_t*)pt_st, (const uint8_t*)zb, (const uint8_t*)yb, n, P, pst);
  B2_TRY(pairing_run(ctx, P, g2_setup_lines(*e), 2, pst, 2 * n, offs, n, f, res, sts, st));
  B2_CUDA(ctx, cudaMemcpyAsync(result, res, n, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(status, sts, n, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

int b200zk_kzg_verify_blob_proof_batch(b200zk_ctx* ctx, uint64_t g2_setup, const uint8_t* blobs, const uint8_t* commitments, const uint8_t* proofs,
                                       size_t n, int* valid) {
  static const char* what = "kzg_verify_blob_proof_batch";
  constexpr size_t kBlob = 4096 * 32;
  if (!ctx || !valid || (n && (!blobs || !commitments || !proofs))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_verify_blob_proof_batch: null argument");
  NvtxRange nvtx("b200zk:kzg_verify_blob_proof_batch");
  DeviceGuard guard(ctx);
  const BasesEntry* e = nullptr;
  B2_TRY(kzg_g2_setup(ctx, g2_setup, what, &e));
  if (!n) { *valid = 1; return B200ZK_OK; }
  cudaStream_t st = ctx->stream;
  uint8_t *d_blobs, *zb, *q, *yb, *in, *pt_st, *rho, *pst, *res, *sts;
  Affine<Fp381>*pts, *P;
  XYZZ<Fp381>* terms;
  F12* f;
  uint32_t* offs;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    d_blobs = c.take<uint8_t>(kBlob * n); zb = c.take<uint8_t>(32 * n); q = c.take<uint8_t>(kBlob * n); yb = c.take<uint8_t>(32 * n);
    in = c.take<uint8_t>(96 * n); pts = c.take<Affine<Fp381>>(2 * n); pt_st = c.take<uint8_t>(2 * n); rho = c.take<uint8_t>(32);
    terms = c.take<XYZZ<Fp381>>(2 * n); P = c.take<Affine<Fp381>>(2); pst = c.take<uint8_t>(2); f = c.take<F12>(2);
    offs = c.take<uint32_t>(2); res = c.take<uint8_t>(1); sts = c.take<uint8_t>(1);
  }));
  char msg[160];
  // 1. every blob element < r (c-kzg blob_to_polynomial): an error, not a false
  B2_CUDA(ctx, cudaMemcpyAsync(d_blobs, blobs, kBlob * n, cudaMemcpyHostToDevice, st));
  B2_TRY(check_blobs(ctx, d_blobs, n, 0, st, what));
  // 2. commitments and proofs: c-kzg validate_kzg_g1 (decompression, subgroup)
  B2_CUDA(ctx, cudaMemcpyAsync(in, commitments, 48 * n, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(in + 48 * n, proofs, 48 * n, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, bls_g1_decode_subgroup, (unsigned)((2 * n + 63) / 64), 64, 0, st, (const uint8_t*)in, 2 * n, pts, pt_st);
  std::vector<uint8_t> h_st(2 * n);
  B2_CUDA(ctx, cudaMemcpyAsync(h_st.data(), pt_st, 2 * n, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  for (size_t k = 0; k < 2 * n; ++k) {
    if (!h_st[k]) continue;
    snprintf(msg, sizeof msg, "%s: the %s of blob %zu %s", what, k < n ? "commitment" : "proof", k % n,
             h_st[k] == B200ZK_ERR_NOT_IN_FIELD ? "has a coordinate >= p" : "has malformed flag bits, is not on the curve or not in the order-r subgroup");
    return fail(ctx, h_st[k], msg);
  }
  // 3. z_i = compute_challenge(blob_i, C_i) on the host; 4. y_i = p_i(z_i) on the device
  std::vector<uint8_t> h_z(32 * n), h_y(32 * n);
  for (size_t b = 0; b < n; ++b) kzg_challenge(blobs + b * kBlob, commitments + 48 * b, &h_z[32 * b]);
  B2_CUDA(ctx, cudaMemcpyAsync(zb, h_z.data(), 32 * n, cudaMemcpyHostToDevice, st));
  B2_TRY(kzg_eval_run(ctx, d_blobs, zb, n, q, yb, st));
  B2_CUDA(ctx, cudaMemcpyAsync(h_y.data(), yb, 32 * n, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  // 5. rho = hash_to_bls_field(SHA-256("RCKZGBATCH___V1_" | 4096 as u64 BE | n as u64 BE | (C_i | z_i | y_i | pi_i) for each i))
  static const uint8_t kDomain[16] = {'R', 'C', 'K', 'Z', 'G', 'B', 'A', 'T', 'C', 'H', '_', '_', '_', 'V', '1', '_'};
  uint8_t lens[16] = {};
  for (int k = 0; k < 8; ++k) { lens[7 - k] = (uint8_t)((uint64_t)4096 >> (8 * k)); lens[15 - k] = (uint8_t)((uint64_t)n >> (8 * k)); }
  Sha256 h;
  h.update(kDomain, 16);
  h.update(lens, 16);
  for (size_t b = 0; b < n; ++b) {
    h.update(commitments + 48 * b, 48);
    h.update(&h_z[32 * b], 32);
    h.update(&h_y[32 * b], 32);
    h.update(proofs + 48 * b, 48);
  }
  uint8_t digest[32], h_rho[32];
  h.final(digest);
  hash_to_bls_field(digest, h_rho);
  // 6. the two random linear combinations; 7. one 2-pair check against (G2, [tau]2)
  const uint32_t h_offs[2] = {0, 2};
  B2_CUDA(ctx, cudaMemcpyAsync(rho, h_rho, 32, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(offs, h_offs, 8, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, kzg_blob_terms, (unsigned)((n + 63) / 64), 64, 0, st, (const Affine<Fp381>*)pts, (const uint8_t*)zb, (const uint8_t*)yb, (const uint8_t*)rho, n, terms);
  B2_LAUNCH(ctx, kzg_blob_fold, 1, 32, 0, st, (const XYZZ<Fp381>*)terms, n, P, pst);
  B2_TRY(pairing_run(ctx, P, g2_setup_lines(*e), 2, pst, 2, offs, 1, f, res, sts, st));
  uint8_t h_res = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(&h_res, res, 1, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  *valid = h_res ? 1 : 0;
  return B200ZK_OK;
}

int b200zk_kzg_verify_cell_proof_batch(b200zk_ctx* ctx, uint64_t g1_setup, uint64_t g2_setup, const uint8_t* blobs, const uint8_t* commitments,
                                       const uint8_t* proofs, size_t n, int* valid) {
  static const char* what = "kzg_verify_cell_proof_batch";
  constexpr size_t kN = 4096, kBlob = kN * 32, kCells = 128, kExt = 2 * kBlob, kCell = kExt / kCells;
  if (!ctx || !valid || (n && (!blobs || !commitments || !proofs))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_verify_cell_proof_batch: null argument");
  NvtxRange nvtx("b200zk:kzg_verify_cell_proof_batch");
  DeviceGuard guard(ctx);
  const BasesEntry *g1 = nullptr, *e = nullptr;
  B2_TRY(cell_setups(ctx, g1_setup, g2_setup, what, &g1, &e));
  if (!n) { *valid = 1; return B200ZK_OK; }
  const size_t m = kCells * n;  // cells and proofs
  cudaStream_t st = ctx->stream;
  uint8_t *d_blobs, *cells, *in, *pt_st, *rbe;
  void *weights, *partial, *s_proof, *s_lin, *s_setup;
  Affine<Fp381>* pts;
  CellTail tail;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    d_blobs = c.take<uint8_t>(kBlob * n); cells = c.take<uint8_t>(kExt * n); in = c.take<uint8_t>(48 * (n + m));
    pts = c.take<Affine<Fp381>>(n + m); pt_st = c.take<uint8_t>(n + m); rbe = c.take<uint8_t>(32);
    weights = c.take<uint4>(2 * 65); partial = c.take<uint4>(2 * 64 * n); s_proof = c.take<uint4>(2 * m); s_lin = c.take<uint4>(2 * (n + m));
    s_setup = c.take<uint4>(2 * kN); tail.take(c);
  }));
  char msg[160];
  // 1. every blob element < r (c-kzg blob_to_polynomial inside compute_cells): an error, not a false
  B2_CUDA(ctx, cudaMemcpyAsync(d_blobs, blobs, kBlob * n, cudaMemcpyHostToDevice, st));
  B2_TRY(check_blobs(ctx, d_blobs, n, 0, st, what));
  // 2. commitments, then proofs: c-kzg validate_kzg_g1 (decompression, subgroup)
  B2_CUDA(ctx, cudaMemcpyAsync(in, commitments, 48 * n, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(in + 48 * n, proofs, 48 * m, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, bls_g1_decode_subgroup, (unsigned)((n + m + 63) / 64), 64, 0, st, (const uint8_t*)in, n + m, pts, pt_st);
  B2_TRY(kzg_cells_run(ctx, d_blobs, n, cells, st));
  std::vector<uint8_t> h_st(n + m), h_cells(kExt * n);
  B2_CUDA(ctx, cudaMemcpyAsync(h_st.data(), pt_st, n + m, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(h_cells.data(), cells, kExt * n, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  for (size_t k = 0; k < n + m; ++k) {
    if (!h_st[k]) continue;
    if (k < n) snprintf(msg, sizeof msg, "%s: the commitment of blob %zu ", what, k);
    else snprintf(msg, sizeof msg, "%s: the proof of blob %zu, cell %zu ", what, (k - n) / kCells, (k - n) % kCells);
    const std::string text = std::string(msg) + (h_st[k] == B200ZK_ERR_NOT_IN_FIELD ? "has a coordinate >= p" : "has malformed flag bits, is not on the curve or not in the order-r subgroup");
    return fail(ctx, h_st[k], text.c_str());
  }
  // 3. r = hash_to_bls_field(SHA-256("RCKZGCBATCH__V1_" | 4096, 64, n, 128 n as u64 BE | the commitments | for each cell:
  //    its commitment index and cell index as u64 BE, its 64 elements, its proof)): the spec's compute_verify_cell_kzg_
  //    proof_batch_challenge, with the commitments listed per blob rather than deduplicated
  static const uint8_t kDomain[16] = {'R', 'C', 'K', 'Z', 'G', 'C', 'B', 'A', 'T', 'C', 'H', '_', '_', 'V', '1', '_'};
  auto put64 = [](uint8_t* o, uint64_t v) { for (int k = 0; k < 8; ++k) o[7 - k] = (uint8_t)(v >> (8 * k)); };
  uint8_t lens[32];
  put64(lens, kN); put64(lens + 8, kCell / 32); put64(lens + 16, n); put64(lens + 24, m);
  Sha256 h;
  h.update(kDomain, 16);
  h.update(lens, 32);
  h.update(commitments, 48 * n);
  for (size_t k = 0; k < m; ++k) {
    uint8_t idx[16];
    put64(idx, k / kCells); put64(idx + 8, k % kCells);
    h.update(idx, 16);
    h.update(&h_cells[(k / kCells) * kExt + (k % kCells) * kCell], kCell);
    h.update(proofs + 48 * k, 48);
  }
  uint8_t digest[32], h_r[32];
  h.final(digest);
  hash_to_bls_field(digest, h_r);
  // 4. the scalars on the device; 5. three MSMs: sum r^k pi_k, the commitments' and r^k h_k^64 pi_k terms, and
  //    [sum r^k I_k(tau)]1 over the Lagrange setup; 6. one 2-pair check against (G2, [tau^64]2)
  B2_CUDA(ctx, cudaMemcpyAsync(rbe, h_r, 32, cudaMemcpyHostToDevice, st));
  B2_TRY(kzg_cell_scalars_run(ctx, d_blobs, n, rbe, weights, partial, s_proof, s_lin, s_setup, st));
  return cell_check_tail(ctx, *g1, *e, pts, n, m, s_proof, s_lin, s_setup, tail, st, valid);
}


int b200zk_kzg_verify_cells(b200zk_ctx* ctx, uint64_t g1_setup, uint64_t g2_setup, const uint8_t* commitments, const uint64_t* cell_indices,
                            const uint8_t* cells, const uint8_t* proofs, size_t n, int* valid) {
  static const char* what = "kzg_verify_cells";
  constexpr size_t kCell = kBatchCellBytes, kElems = kBatchCellN;
  if (!ctx || !valid || (n && (!commitments || !cell_indices || !cells || !proofs))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_verify_cells: null argument");
  NvtxRange nvtx("b200zk:kzg_verify_cells");
  DeviceGuard guard(ctx);
  const BasesEntry *g1 = nullptr, *e = nullptr;
  B2_TRY(cell_setups(ctx, g1_setup, g2_setup, what, &g1, &e));
  if (!n) { *valid = 1; return B200ZK_OK; }
  char msg[192];
  // 1. cell indices < 128, then the deduplicated commitments and the groupings by commitment and by cell index (host)
  CellBatch b;
  const size_t bad_index = cell_batch_build(commitments, cell_indices, n, &b);
  if (bad_index < n) {
    snprintf(msg, sizeof msg, "%s: cell %zu: index %llu is not below 128", what, bad_index, (unsigned long long)cell_indices[bad_index]);
    return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, msg);
  }
  const size_t u = b.unique.size(), n_cols = b.columns.size();
  std::vector<uint8_t> h_commit(48 * u);
  for (size_t i = 0; i < u; ++i) memcpy(&h_commit[48 * i], commitments + 48 * (size_t)b.unique[i], 48);
  // meta: idx (n) | commit_off (u + 1) | by_commit (n) | column_off (n_cols + 1) | by_column (n) | columns (n_cols)
  std::vector<uint32_t> meta;
  meta.reserve(3 * n + u + 2 * n_cols + 2);
  for (size_t k = 0; k < n; ++k) meta.push_back((uint32_t)cell_indices[k]);
  for (const std::vector<uint32_t>* v : {&b.commit_off, &b.by_commit, &b.column_off, &b.by_column, &b.columns}) meta.insert(meta.end(), v->begin(), v->end());
  cudaStream_t st = ctx->stream;
  uint8_t *in, *d_cells, *pt_st, *rbe;
  uint32_t* d_meta;
  unsigned long long* d_bad;
  void *rpow, *partial, *s_proof, *s_lin, *s_setup;
  Affine<Fp381>* pts;
  CellTail tail;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    in = c.take<uint8_t>(48 * (u + n)); d_cells = c.take<uint8_t>(kCell * n); d_meta = c.take<uint32_t>(meta.size()); d_bad = c.take<unsigned long long>(1);
    pts = c.take<Affine<Fp381>>(u + n); pt_st = c.take<uint8_t>(u + n); rbe = c.take<uint8_t>(32);
    rpow = c.take<uint4>(2 * n); partial = c.take<uint4>(2 * kElems * n_cols); s_proof = c.take<uint4>(2 * n); s_lin = c.take<uint4>(2 * (u + n));
    s_setup = c.take<uint4>(2 * 4096); tail.take(c);
  }));
  VCellsMeta vm;
  vm.n = n; vm.n_commit = u; vm.n_cols = n_cols;
  vm.idx = d_meta; vm.commit_off = vm.idx + n; vm.by_commit = vm.commit_off + u + 1;
  vm.column_off = vm.by_commit + n; vm.by_column = vm.column_off + n_cols + 1; vm.columns = vm.by_column + n;
  // 2. enqueue the inputs, the decompression and subgroup checks of the deduplicated commitments and the proofs
  //    (c-kzg validate_kzg_g1), and the range check of every cell element
  const unsigned long long h_bad = kElems * n;
  B2_CUDA(ctx, cudaMemcpyAsync(in, h_commit.data(), 48 * u, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(in + 48 * u, proofs, 48 * n, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(d_meta, meta.data(), 4 * meta.size(), cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(d_bad, &h_bad, 8, cudaMemcpyHostToDevice, st));
  // every copy before the first kernel: a copy from pageable memory queued behind the subgroup checks would hold the
  // host until they finish, and the hash with it
  B2_CUDA(ctx, cudaMemcpyAsync(d_cells, cells, kCell * n, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, bls_g1_decode_subgroup, (unsigned)((u + n + 63) / 64), 64, 0, st, (const uint8_t*)in, u + n, pts, pt_st);
  B2_TRY(bls_scalars_check_enqueue(ctx, d_cells, kElems * n, true, st, d_bad));
  // 3. while they run: r = compute_verify_cell_kzg_proof_batch_challenge over the caller's buffers (host SHA-256)
  uint8_t h_r[32];
  cell_batch_challenge(b, commitments, cell_indices, cells, proofs, h_r);
  // 4. the statuses, in the spec's order: the deduplicated commitments, the cell elements, the proofs
  std::vector<uint8_t> h_st(u + n);
  unsigned long long h_bad_out = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(h_st.data(), pt_st, u + n, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(&h_bad_out, d_bad, 8, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  auto point_error = [&](size_t p) {
    if (p < u) snprintf(msg, sizeof msg, "%s: the commitment of cell %u ", what, b.unique[p]);
    else snprintf(msg, sizeof msg, "%s: the proof of cell %zu ", what, p - u);
    const std::string text = std::string(msg) + (h_st[p] == B200ZK_ERR_NOT_IN_FIELD ? "has a coordinate >= p" : "has malformed flag bits, is not on the curve or not in the order-r subgroup");
    return fail(ctx, h_st[p], text.c_str());
  };
  for (size_t p = 0; p < u; ++p)
    if (h_st[p]) return point_error(p);
  if (h_bad_out < kElems * n) {
    snprintf(msg, sizeof msg, "%s: cell %llu, element %llu is >= the BLS12-381 group order", what, h_bad_out / kElems, h_bad_out % kElems);
    return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, msg);
  }
  for (size_t p = u; p < u + n; ++p)
    if (h_st[p]) return point_error(p);
  // 5. the scalars on the device (r^k, the commitment weights, the per-column interpolation); 6. the shared tail
  B2_CUDA(ctx, cudaMemcpyAsync(rbe, h_r, 32, cudaMemcpyHostToDevice, st));
  B2_TRY(kzg_vcells_scalars_run(ctx, d_cells, vm, rbe, rpow, partial, s_proof, s_lin, s_setup, st));
  return cell_check_tail(ctx, *g1, *e, pts, u, n, s_proof, s_lin, s_setup, tail, st, valid);
}

}  // extern "C"
