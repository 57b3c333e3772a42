// bls_pairing.cu -- the BLS12-381 pairing on the device and the three calls of the reference that rest on it:
//   the EIP-2537 pairing check        Crypto::bls12_381_pairing_check, /root/reference/crates/common/crypto/provider.rs:642-672
//   verify_kzg_proof (0x0a precompile) Crypto::verify_kzg_proof, provider.rs:463-507 (levm precompiles.rs:923-985)
//   verify_blob_kzg_proof_batch        BlobsBundle::verify_kzg_proofs -> kzg::verify_kzg_proof_batch (blobs_bundle.rs:155-173,
//                                      kzg.rs:168-192); verify_blob_kzg_proof (provider.rs:509-544) is its batch of one
//
// Tower: Fp2 = Fp[u]/(u^2 + 1) (bls12.cuh), Fp6 = Fp2[v]/(v^3 - (1 + u)), Fp12 = Fp6[w]/(w^2 - v).  The twist is M-type:
// E': y^2 = x^3 + 4(1 + u).
// Miller loop: optimal ate over |x| = 0xd201000000010000 (64 bits: 63 doublings, 5 additions).  The line coefficients of a
// G2 point depend on that point only, so a prepare pass (one thread per G2 point) writes its 68 triples in homogeneous
// projective coordinates -- no inversion anywhere -- and the Miller kernel (one thread per pair) only evaluates them at P:
// the G2Prepared + multi_miller_loop split of provider.rs:651-670.  x is negative: f is conjugated at the end.
// Final exponentiation: the easy part f^((p^6 - 1)(p^2 + 1)) (conjugate, one inversion, one p^2 Frobenius), then the hard
// part through the x-chain 3 (p^4 - p^2 + 1)/r = (x - 1)^2 (x + p) (x^2 + p^2 - 1) + 3: five exponentiations by x, three
// Frobenius maps and a handful of products instead of a generic 1269-bit power.  It yields the CUBE of the reduced pairing;
// a check asks whether a product of pairings is one, and since gcd(3, r) = 1, z^3 = 1 exactly when z = 1 for z in the
// order-r group mu_r.  tests/test_bls12_pairing_host.py recomputes every constant of this file and checks the identity.
#include "bls12.cuh"
#include "sha256.h"
#include <cstring>
#include <vector>

namespace b200zk {
namespace {

typedef Fp2_381 F2;

// xi^(k (p - 1) / 6), xi = 1 + u, k = 0..5 (c0, c1): the p-power Frobenius of the coefficient of w^k; canonical limbs
__constant__ uint32_t kFrob1[6][2][12] = {
    {{0x00000001u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u},
     {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
    {{0x92235fb8u, 0x8d0775edu, 0x63e7813du, 0xf67ea53du, 0x84bab9c4u, 0x7b2443d7u, 0x3cbd5f4fu, 0x0fd603fdu, 0x202c0d1fu, 0xc231beb4u, 0x02bb0667u, 0x1904d3bfu},
     {0x6ddc4af3u, 0x2cf78a12u, 0x4d6c7ec2u, 0x282d5ac1u, 0x71f63c5fu, 0xec0c8ec9u, 0xb6c7b36fu, 0x54a14787u, 0x231f9fb8u, 0x88e9e902u, 0x36c4e032u, 0x00fc3e2bu}},
    {{0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u},
     {0x0000aaacu, 0x8bfd0000u, 0x4f49fffdu, 0x409427ebu, 0x0fb85f9bu, 0x897d2965u, 0x89759ad4u, 0xaa0d857du, 0x63d4de85u, 0xec024086u, 0x397fe699u, 0x1a0111eau}},
    {{0xede3cc09u, 0xc81084fbu, 0x72ec05f4u, 0xee67992fu, 0x009241c5u, 0x77f76e17u, 0xc2d3435eu, 0x48395dabu, 0x6bd17ffeu, 0x6831e36du, 0x37ff400bu, 0x06af0e04u},
     {0xede3cc09u, 0xc81084fbu, 0x72ec05f4u, 0xee67992fu, 0x009241c5u, 0x77f76e17u, 0xc2d3435eu, 0x48395dabu, 0x6bd17ffeu, 0x6831e36du, 0x37ff400bu, 0x06af0e04u}},
    {{0x0000aaadu, 0x8bfd0000u, 0x4f49fffdu, 0x409427ebu, 0x0fb85f9bu, 0x897d2965u, 0x89759ad4u, 0xaa0d857du, 0x63d4de85u, 0xec024086u, 0x397fe699u, 0x1a0111eau},
     {0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u}},
    {{0x80078116u, 0x9b18fae9u, 0x257f8732u, 0xc63a3e6eu, 0x8e9c0566u, 0x8beadf4du, 0x0c0b8feeu, 0xf3981624u, 0x48b1e045u, 0xdf47fa6bu, 0x013a5fd8u, 0x05b2cfd9u},
     {0x7ff82995u, 0x1ee60516u, 0x8bd478cdu, 0x5871c190u, 0x6814f0bdu, 0xdb45f353u, 0xe77982d0u, 0x70df3560u, 0xfa99cc91u, 0x6bd3ad4au, 0x384586c1u, 0x144e4211u}},
};
// xi^(k (p^2 - 1) / 6), k = 0..5: the p^2-power Frobenius (all six lie in Fp); canonical limbs
__constant__ uint32_t kFrob2[6][12] = {
    {0x00000001u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000000u},
    {0xfffeffffu, 0x2e01ffffu, 0x620a0002u, 0xde17d813u, 0xe6f89688u, 0xddb3a93bu, 0x6a0f77eau, 0xba69c607u, 0xdf76ce51u, 0x5f19672fu, 0x00000000u, 0x00000000u},
    {0xfffefffeu, 0x2e01ffffu, 0x620a0002u, 0xde17d813u, 0xe6f89688u, 0xddb3a93bu, 0x6a0f77eau, 0xba69c607u, 0xdf76ce51u, 0x5f19672fu, 0x00000000u, 0x00000000u},
    {0xffffaaaau, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau},
    {0x0000aaacu, 0x8bfd0000u, 0x4f49fffdu, 0x409427ebu, 0x0fb85f9bu, 0x897d2965u, 0x89759ad4u, 0xaa0d857du, 0x63d4de85u, 0xec024086u, 0x397fe699u, 0x1a0111eau},
    {0x0000aaadu, 0x8bfd0000u, 0x4f49fffdu, 0x409427ebu, 0x0fb85f9bu, 0x897d2965u, 0x89759ad4u, 0xaa0d857du, 0x63d4de85u, 0xec024086u, 0x397fe699u, 0x1a0111eau},
};
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

constexpr uint64_t kX = 0xd201000000010000ull;  // |x|; x = -|x|
constexpr int kLines = 68;                      // line triples per G2 point: 63 doublings + 5 additions
constexpr uint8_t kTrivial = 0x80;              // pair status bit: a side is the identity, the pair contributes 1

struct Fp6b { F2 c0, c1, c2; };
struct Fp12b { Fp6b c0, c1; };
struct BlsLine { F2 c0, c1, c2; };  // l = c0 + (c1 xP) v + (c2 yP) v w  (mul_by_014 positions)

B2_D Fp381 fp_const(const uint32_t* canonical) {
  Fp381 a;
#pragma unroll
  for (int k = 0; k < 12; ++k) a.v[k] = canonical[k];
  return Fp381::to_mont(a);
}

// ---- Fp6 ------------------------------------------------------------------------------------------------------------
B2_D Fp6b f6_zero() { return {F2::zero(), F2::zero(), F2::zero()}; }
B2_D Fp6b f6_one() { return {F2::one(), F2::zero(), F2::zero()}; }
B2_D Fp6b f6_add(const Fp6b& a, const Fp6b& b) { return {F2::add(a.c0, b.c0), F2::add(a.c1, b.c1), F2::add(a.c2, b.c2)}; }
B2_D Fp6b f6_sub(const Fp6b& a, const Fp6b& b) { return {F2::sub(a.c0, b.c0), F2::sub(a.c1, b.c1), F2::sub(a.c2, b.c2)}; }
B2_D Fp6b f6_neg(const Fp6b& a) { return {F2::neg(a.c0), F2::neg(a.c1), F2::neg(a.c2)}; }
B2_D Fp6b f6_mul_v(const Fp6b& a) { return {F2::mul_xi(a.c2), a.c0, a.c1}; }
__device__ __noinline__ Fp6b f6_mul(const Fp6b& a, const Fp6b& b) {  // Karatsuba over Fp2: six products
  const F2 t0 = F2::mul(a.c0, b.c0), t1 = F2::mul(a.c1, b.c1), t2 = F2::mul(a.c2, b.c2);
  Fp6b r;
  r.c0 = F2::add(t0, F2::mul_xi(F2::sub(F2::sub(F2::mul(F2::add(a.c1, a.c2), F2::add(b.c1, b.c2)), t1), t2)));
  r.c1 = F2::add(F2::sub(F2::sub(F2::mul(F2::add(a.c0, a.c1), F2::add(b.c0, b.c1)), t0), t1), F2::mul_xi(t2));
  r.c2 = F2::add(F2::sub(F2::sub(F2::mul(F2::add(a.c0, a.c2), F2::add(b.c0, b.c2)), t0), t2), t1);
  return r;
}
// a (b0 + b1 v): the line's sparse shape
__device__ __noinline__ Fp6b f6_mul_01(const Fp6b& a, const F2& b0, const F2& b1) {
  return {F2::add(F2::mul(a.c0, b0), F2::mul_xi(F2::mul(a.c2, b1))), F2::add(F2::mul(a.c0, b1), F2::mul(a.c1, b0)),
          F2::add(F2::mul(a.c1, b1), F2::mul(a.c2, b0))};
}
B2_D Fp6b f6_mul_1(const Fp6b& a, const F2& b1) { return {F2::mul_xi(F2::mul(a.c2, b1)), F2::mul(a.c0, b1), F2::mul(a.c1, b1)}; }
__device__ __noinline__ Fp6b f6_inv(const Fp6b& a) {
  const F2 A = F2::sub(F2::sqr(a.c0), F2::mul_xi(F2::mul(a.c1, a.c2)));
  const F2 B = F2::sub(F2::mul_xi(F2::sqr(a.c2)), F2::mul(a.c0, a.c1));
  const F2 C = F2::sub(F2::sqr(a.c1), F2::mul(a.c0, a.c2));
  const F2 Fi = F2::inv(F2::add(F2::mul(a.c0, A), F2::mul_xi(F2::add(F2::mul(a.c2, B), F2::mul(a.c1, C)))));
  return {F2::mul(A, Fi), F2::mul(B, Fi), F2::mul(C, Fi)};
}

// ---- Fp12 -----------------------------------------------------------------------------------------------------------
B2_D Fp12b f12_one() { return {f6_one(), f6_zero()}; }
__device__ __noinline__ Fp12b f12_mul(const Fp12b& a, const Fp12b& b) {
  const Fp6b t0 = f6_mul(a.c0, b.c0), t1 = f6_mul(a.c1, b.c1);
  return {f6_add(t0, f6_mul_v(t1)), f6_sub(f6_sub(f6_mul(f6_add(a.c0, a.c1), f6_add(b.c0, b.c1)), t0), t1)};
}
__device__ __noinline__ Fp12b f12_sqr(const Fp12b& a) {  // complex squaring: two Fp6 products
  const Fp6b ab = f6_mul(a.c0, a.c1);
  const Fp6b c0 = f6_sub(f6_sub(f6_mul(f6_add(a.c0, a.c1), f6_add(a.c0, f6_mul_v(a.c1))), ab), f6_mul_v(ab));
  return {c0, f6_add(ab, ab)};
}
// f (c0 + c1 v + c4 v w): aa = f.c0 (c0 + c1 v), bb = f.c1 (c4 v), then Karatsuba over Fp6
__device__ __noinline__ Fp12b f12_mul_014(const Fp12b& f, const F2& c0, const F2& c1, const F2& c4) {
  const Fp6b aa = f6_mul_01(f.c0, c0, c1), bb = f6_mul_1(f.c1, c4);
  const Fp6b t = f6_mul_01(f6_add(f.c0, f.c1), c0, F2::add(c1, c4));
  return {f6_add(aa, f6_mul_v(bb)), f6_sub(f6_sub(t, aa), bb)};
}
B2_D Fp12b f12_conj(const Fp12b& a) { return {a.c0, f6_neg(a.c1)}; }
__device__ __noinline__ Fp12b f12_inv(const Fp12b& a) {
  const Fp6b t = f6_inv(f6_sub(f6_mul(a.c0, a.c0), f6_mul_v(f6_mul(a.c1, a.c1))));
  return {f6_mul(a.c0, t), f6_neg(f6_mul(a.c1, t))};
}
B2_D bool f12_is_one(const Fp12b& a) {
  return a.c0.c0 == F2::one() && a.c0.c1.is_zero() && a.c0.c2.is_zero() && a.c1.c0.is_zero() && a.c1.c1.is_zero() && a.c1.c2.is_zero();
}
// (sum_k a_k w^k)^p = sum_k conj(a_k) xi^(k (p-1)/6) w^k; the coefficient of w^k is c0.c_(k/2) for even k, c1.c_(k/2) for odd
B2_D F2 frob1_coeff(int k) { return {fp_const(kFrob1[k][0]), fp_const(kFrob1[k][1])}; }
__device__ __noinline__ Fp12b f12_frob(const Fp12b& a) {
  return {{F2::mul(F2::conj(a.c0.c0), frob1_coeff(0)), F2::mul(F2::conj(a.c0.c1), frob1_coeff(2)), F2::mul(F2::conj(a.c0.c2), frob1_coeff(4))},
          {F2::mul(F2::conj(a.c1.c0), frob1_coeff(1)), F2::mul(F2::conj(a.c1.c1), frob1_coeff(3)), F2::mul(F2::conj(a.c1.c2), frob1_coeff(5))}};
}
__device__ __noinline__ Fp12b f12_frob2(const Fp12b& a) {  // Fp2 is fixed by the p^2 power: only the w^k factors move
  return {{a.c0.c0, F2::scale(a.c0.c1, fp_const(kFrob2[2])), F2::scale(a.c0.c2, fp_const(kFrob2[4]))},
          {F2::scale(a.c1.c0, fp_const(kFrob2[1])), F2::scale(a.c1.c1, fp_const(kFrob2[3])), F2::scale(a.c1.c2, fp_const(kFrob2[5]))}};
}

// f^x for f in the cyclotomic subgroup (there f^-1 = conj f): square-and-multiply over |x|, then conjugate
__device__ __noinline__ Fp12b f12_exp_x(const Fp12b& f) {
  Fp12b acc = f;
#pragma unroll 1
  for (int i = 62; i >= 0; --i) {
    acc = f12_sqr(acc);
    if ((kX >> i) & 1) acc = f12_mul(acc, f);
  }
  return f12_conj(acc);
}

// f^(3 (p^12 - 1)/r): see the header for why the cube answers "is the pairing product one" exactly
__device__ __noinline__ Fp12b final_exponentiate(const Fp12b& f0) {
  Fp12b f = f12_mul(f12_conj(f0), f12_inv(f0));  // f^(p^6 - 1)
  f = f12_mul(f12_frob2(f), f);                   // ^(p^2 + 1): f is now in the cyclotomic subgroup
  Fp12b t = f12_mul(f12_exp_x(f), f12_conj(f));   // f^(x - 1)
  t = f12_mul(f12_exp_x(t), f12_conj(t));         // f^((x - 1)^2)
  t = f12_mul(f12_exp_x(t), f12_frob(t));         // ^(x + p)
  t = f12_mul(f12_mul(f12_exp_x(f12_exp_x(t)), f12_frob2(t)), f12_conj(t));  // ^(x^2 + p^2 - 1)
  return f12_mul(t, f12_mul(f12_sqr(f), f));      // * f^3
}

// ---- G2 line coefficients, homogeneous projective T = (X : Y : Z), M-type twist ---------------------------------------
struct G2Proj { F2 x, y, z; };

B2_D F2 mul_b2(const F2& a) { return F2::dbl(F2::dbl(F2::mul_xi(a))); }  // * 4 (1 + u)

// T = 2T; line through the tangent (Costello-Lange-Naehrig 2010, as arkworks' bls12 G2Prepared)
B2_D BlsLine line_double(G2Proj& T, const Fp381& two_inv) {
  const F2 a = F2::scale(F2::mul(T.x, T.y), two_inv), b = F2::sqr(T.y), c = F2::sqr(T.z);
  const F2 e = mul_b2(F2::add(F2::dbl(c), c)), f = F2::add(F2::dbl(e), e);
  const F2 g = F2::scale(F2::add(b, f), two_inv);
  const F2 h = F2::sub(F2::sqr(F2::add(T.y, T.z)), F2::add(b, c));
  const F2 i = F2::sub(e, b), j = F2::sqr(T.x), e2 = F2::sqr(e);
  T.x = F2::mul(a, F2::sub(b, f));
  T.y = F2::sub(F2::sqr(g), F2::add(F2::dbl(e2), e2));
  T.z = F2::mul(b, h);
  return {i, F2::add(F2::dbl(j), j), F2::neg(h)};
}

// T = T + Q; line through T and Q
B2_D BlsLine line_add(G2Proj& T, const Affine<F2>& q) {
  const F2 theta = F2::sub(T.y, F2::mul(q.y, T.z)), lambda = F2::sub(T.x, F2::mul(q.x, T.z));
  const F2 c = F2::sqr(theta), d = F2::sqr(lambda), e = F2::mul(lambda, d), f = F2::mul(T.z, c), g = F2::mul(T.x, d);
  const F2 h = F2::sub(F2::add(e, f), F2::dbl(g));
  T.x = F2::mul(lambda, h);
  T.y = F2::sub(F2::mul(theta, F2::sub(g, h)), F2::mul(e, T.y));
  T.z = F2::mul(T.z, e);
  return {F2::sub(F2::mul(theta, q.x), F2::mul(lambda, q.y)), F2::neg(theta), lambda};
}

__device__ __noinline__ void g2_prepare(const Affine<F2>& q, BlsLine* out) {
  Fp381 two_inv = fp381_half();  // (p + 1)/2 = (p - 1)/2 + 1; limb 0 of (p - 1)/2 is 0xffffd555: no carry
  two_inv.v[0] += 1;
  two_inv = Fp381::to_mont(two_inv);
  G2Proj T = {q.x, q.y, F2::one()};
  int k = 0;
#pragma unroll 1
  for (int i = 62; i >= 0; --i) {
    out[k++] = line_double(T, two_inv);
    if ((kX >> i) & 1) out[k++] = line_add(T, q);
  }
}

// f_{|x|,Q}(P) over prepared lines, conjugated for x < 0
__device__ __noinline__ Fp12b miller_prepared(const BlsLine* L, const Affine<Fp381>& p) {
  Fp12b f = f12_one();
  int k = 0;
#pragma unroll 1
  for (int i = 62; i >= 0; --i) {
    f = f12_sqr(f);
    BlsLine l = L[k++];
    f = f12_mul_014(f, l.c0, F2::scale(l.c1, p.x), F2::scale(l.c2, p.y));
    if ((kX >> i) & 1) {
      l = L[k++];
      f = f12_mul_014(f, l.c0, F2::scale(l.c1, p.x), F2::scale(l.c2, p.y));
    }
  }
  return f12_conj(f);
}

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
    else if ((!p.is_inf() && !g1_in_subgroup(p)) || (!q.is_inf() && !g2_in_subgroup(q))) s = B200ZK_ERR_NOT_ON_CURVE;
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
      if (!g2_in_subgroup(pt)) bad_point = true;
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
__global__ void __launch_bounds__(32) bls_miller(const Affine<Fp381>* P, const BlsLine* lines, uint32_t period, const uint8_t* pst, size_t n, Fp12b* f) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Fp12b r = f12_one();
  if (!pst[i]) r = miller_prepared(lines + kLines * (period ? i % period : i), P[i]);
  f[i] = r;
}

// one thread per check: the product of its Miller values, one final exponentiation.  A range error anywhere in the check
// outranks a curve error (every point is range-checked before any curve check)
__global__ void __launch_bounds__(32) bls_pairing_final(const Fp12b* f, const uint8_t* pst, const uint32_t* offsets, size_t count, uint8_t* result, uint8_t* status) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= count) return;
  const uint32_t lo = offsets[i], hi = offsets[i + 1];
  uint32_t s = 0;
  for (uint32_t k = lo; k < hi; ++k) {
    const uint32_t ps = pst[k] & ~kTrivial;
    if (ps == B200ZK_ERR_NOT_IN_FIELD) s = ps;
    else if (ps && !s) s = ps;
  }
  uint32_t ok = 0;
  if (!s) {
    Fp12b acc = f12_one();
    for (uint32_t k = lo; k < hi; ++k) acc = f12_mul(acc, f[k]);
    ok = f12_is_one(final_exponentiate(acc)) ? 1u : 0u;
  }
  result[i] = (uint8_t)ok;
  status[i] = (uint8_t)s;
}

// c-kzg validate_kzg_g1 on 48-byte compressed points: decompression (status 2 / 3) and r P = O (status 3); identity valid
__global__ void __launch_bounds__(64) bls_g1_decode_subgroup(const uint8_t* __restrict__ in, size_t n, Affine<Fp381>* out, uint8_t* st) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<Fp381> p;
  uint32_t s = bls_g1_decompress(in + 48 * i, &p);
  if (!s && !p.is_inf() && !g1_in_subgroup(p)) s = B200ZK_ERR_NOT_ON_CURVE;
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
                const uint32_t* offsets, size_t count, Fp12b* f, uint8_t* result, uint8_t* status, cudaStream_t st) {
  if (n_pairs) B2_LAUNCH(ctx, bls_miller, (unsigned)((n_pairs + 31) / 32), 32, 0, st, P, lines, period, pst, n_pairs, f);
  B2_LAUNCH(ctx, bls_pairing_final, (unsigned)((count + 31) / 32), 32, 0, st, (const Fp12b*)f, pst, offsets, count, result, status);
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
  Fp12b* f;
  uint32_t* offs;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    in = c.take<uint8_t>(384 * n); P = c.take<Affine<Fp381>>(n); Q = c.take<Affine<F2>>(n); pst = c.take<uint8_t>(n);
    lines = c.take<BlsLine>(kLines * n); f = c.take<Fp12b>(n); offs = c.take<uint32_t>(count + 1); res = c.take<uint8_t>(count); sts = c.take<uint8_t>(count);
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
  Fp12b* f;
  uint32_t* offs;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    in = c.take<uint8_t>(96 * n); zb = c.take<uint8_t>(32 * n); yb = c.take<uint8_t>(32 * n); pts = c.take<Affine<Fp381>>(2 * n);
    pt_st = c.take<uint8_t>(2 * n); P = c.take<Affine<Fp381>>(2 * n); pst = c.take<uint8_t>(2 * n); f = c.take<Fp12b>(2 * n);
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
  Fp12b* f;
  uint32_t* offs;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    d_blobs = c.take<uint8_t>(kBlob * n); zb = c.take<uint8_t>(32 * n); q = c.take<uint8_t>(kBlob * n); yb = c.take<uint8_t>(32 * n);
    in = c.take<uint8_t>(96 * n); pts = c.take<Affine<Fp381>>(2 * n); pt_st = c.take<uint8_t>(2 * n); rho = c.take<uint8_t>(32);
    terms = c.take<XYZZ<Fp381>>(2 * n); P = c.take<Affine<Fp381>>(2); pst = c.take<uint8_t>(2); f = c.take<Fp12b>(2);
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
  const BasesEntry* g1 = find_bases(ctx, g1_setup, Group::Bls12G1, "kzg_verify_cell_proof_batch: unknown G1 setup handle");
  if (!g1) return B200ZK_ERR_INVALID_ARG;
  if (g1->n != kN) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_verify_cell_proof_batch: the G1 setup must hold FIELD_ELEMENTS_PER_BLOB = 4096 points");
  const BasesEntry* e = nullptr;
  B2_TRY(kzg_g2_setup(ctx, g2_setup, what, &e));
  if (e->n < 65) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_verify_cell_proof_batch: the G2 setup must hold at least 65 points ([tau^64]2 is point 64)");
  if (!n) { *valid = 1; return B200ZK_OK; }
  const size_t m = kCells * n;  // cells and proofs
  cudaStream_t st = ctx->stream;
  uint8_t *d_blobs, *cells, *in, *pt_st, *rbe, *pst, *res, *sts;
  void *weights, *partial, *s_proof, *s_lin, *s_setup;
  Affine<Fp381>*pts, *P;
  Affine<F2>* q2;
  XYZZ<Fp381>* parts;
  BlsLine* lines;
  Fp12b* f;
  uint32_t* offs;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    d_blobs = c.take<uint8_t>(kBlob * n); cells = c.take<uint8_t>(kExt * n); in = c.take<uint8_t>(48 * (n + m));
    pts = c.take<Affine<Fp381>>(n + m); pt_st = c.take<uint8_t>(n + m); rbe = c.take<uint8_t>(32);
    weights = c.take<uint4>(2 * 65); partial = c.take<uint4>(2 * 64 * n); s_proof = c.take<uint4>(2 * m); s_lin = c.take<uint4>(2 * (n + m));
    s_setup = c.take<uint4>(2 * kN); parts = c.take<XYZZ<Fp381>>(3); q2 = c.take<Affine<F2>>(2); lines = c.take<BlsLine>(2 * kLines);
    P = c.take<Affine<Fp381>>(2); pst = c.take<uint8_t>(2); f = c.take<Fp12b>(2); offs = c.take<uint32_t>(2); res = c.take<uint8_t>(1); sts = c.take<uint8_t>(1);
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
  B2_TRY(msm_run_bls(ctx, pts + n, s_proof, m, 0, st, parts));
  B2_TRY(msm_run_bls(ctx, pts, s_lin, n + m, 0, st, parts + 1));
  B2_TRY(msm_run_bls(ctx, g1->d.p, s_setup, kN, 0, st, parts + 2, g1->table_c, g1->n));
  B2_LAUNCH(ctx, kzg_cell_fold, 1, 32, 0, st, (const XYZZ<Fp381>*)parts, P, pst);
  const Affine<F2>* g2pts = (const Affine<F2>*)e->d.p;
  B2_CUDA(ctx, cudaMemcpyAsync(q2, g2pts, sizeof(Affine<F2>), cudaMemcpyDeviceToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(q2 + 1, g2pts + 64, sizeof(Affine<F2>), cudaMemcpyDeviceToDevice, st));
  B2_LAUNCH(ctx, bls_g2_prepare, 1, 64, 0, st, (const Affine<F2>*)q2, (const uint8_t*)nullptr, (size_t)2, lines);
  const uint32_t h_offs[2] = {0, 2};
  B2_CUDA(ctx, cudaMemcpyAsync(offs, h_offs, 8, cudaMemcpyHostToDevice, st));
  B2_TRY(pairing_run(ctx, P, lines, 2, pst, 2, offs, 1, f, res, sts, st));
  uint8_t h_res = 0;
  B2_CUDA(ctx, cudaMemcpyAsync(&h_res, res, 1, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  *valid = h_res ? 1 : 0;
  return B200ZK_OK;
}

}  // extern "C"
