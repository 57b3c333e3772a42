// bls_pairing.cuh -- the stages of the BLS12-381 optimal ate pairing: Frobenius maps, the exponentiation by x, the final
// exponentiation, the G2 line coefficients and the Miller loop over prepared lines.  bls_pairing.cu builds its kernels on
// them; tests/csrc/pairing_conformance.cu runs each stage alone.  See bls_pairing.cu for the algorithm.
// Internal linkage (anonymous namespace, __constant__ tables): the build has no -rdc, so each translation unit that
// includes this header holds its own copy.
#pragma once
#include "bls12.cuh"
#include "tower.cuh"

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

constexpr uint64_t kX = 0xd201000000010000ull;  // |x|; x = -|x|
constexpr int kLines = 68;                      // line triples per G2 point: 63 doublings + 5 additions

typedef Fp12<F2> F12;
struct BlsLine { F2 c0, c1, c2; };  // l = c0 + (c1 xP) v + (c2 yP) v w  (mul_by_014 positions)

B2_D Fp381 fp_const(const uint32_t* canonical) {
  Fp381 a;
#pragma unroll
  for (int k = 0; k < 12; ++k) a.v[k] = canonical[k];
  return Fp381::to_mont(a);
}

// ---- Frobenius maps -------------------------------------------------------------------------------------------------
// (sum_k a_k w^k)^p = sum_k conj(a_k) xi^(k (p-1)/6) w^k; the coefficient of w^k is c0.c_(k/2) for even k, c1.c_(k/2) for odd
B2_D F2 frob1_coeff(int k) { return {fp_const(kFrob1[k][0]), fp_const(kFrob1[k][1])}; }
__device__ __noinline__ F12 f12_frob(const F12& a) {
  return {{F2::mul(F2::conj(a.c0.c0), frob1_coeff(0)), F2::mul(F2::conj(a.c0.c1), frob1_coeff(2)), F2::mul(F2::conj(a.c0.c2), frob1_coeff(4))},
          {F2::mul(F2::conj(a.c1.c0), frob1_coeff(1)), F2::mul(F2::conj(a.c1.c1), frob1_coeff(3)), F2::mul(F2::conj(a.c1.c2), frob1_coeff(5))}};
}
__device__ __noinline__ F12 f12_frob2(const F12& a) {  // Fp2 is fixed by the p^2 power: only the w^k factors move
  return {{a.c0.c0, F2::scale(a.c0.c1, fp_const(kFrob2[2])), F2::scale(a.c0.c2, fp_const(kFrob2[4]))},
          {F2::scale(a.c1.c0, fp_const(kFrob2[1])), F2::scale(a.c1.c1, fp_const(kFrob2[3])), F2::scale(a.c1.c2, fp_const(kFrob2[5]))}};
}

// f^x for f in the cyclotomic subgroup (there f^-1 = conj f): square-and-multiply over |x|, then conjugate
__device__ __noinline__ F12 f12_exp_x(const F12& f) {
  F12 acc = f;
#pragma unroll 1
  for (int i = 62; i >= 0; --i) {
    acc = F12::sqr(acc);
    if ((kX >> i) & 1) acc = F12::mul(acc, f);
  }
  return F12::conj(acc);
}

// f^(3 (p^12 - 1)/r): see the header for why the cube answers "is the pairing product one" exactly
__device__ __noinline__ F12 final_exponentiate(const F12& f0) {
  F12 f = F12::mul(F12::conj(f0), F12::inv(f0));  // f^(p^6 - 1)
  f = F12::mul(f12_frob2(f), f);                   // ^(p^2 + 1): f is now in the cyclotomic subgroup
  F12 t = F12::mul(f12_exp_x(f), F12::conj(f));    // f^(x - 1)
  t = F12::mul(f12_exp_x(t), F12::conj(t));        // f^((x - 1)^2)
  t = F12::mul(f12_exp_x(t), f12_frob(t));         // ^(x + p)
  t = F12::mul(F12::mul(f12_exp_x(f12_exp_x(t)), f12_frob2(t)), F12::conj(t));  // ^(x^2 + p^2 - 1)
  return F12::mul(t, F12::mul(F12::sqr(f), f));   // * f^3
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
__device__ __noinline__ F12 miller_prepared(const BlsLine* L, const Affine<Fp381>& p) {
  F12 f = F12::one();
  int k = 0;
#pragma unroll 1
  for (int i = 62; i >= 0; --i) {
    f = F12::sqr(f);
    BlsLine l = L[k++];
    f = F12::mul_014(f, l.c0, F2::scale(l.c1, p.x), F2::scale(l.c2, p.y));
    if ((kX >> i) & 1) {
      l = L[k++];
      f = F12::mul_014(f, l.c0, F2::scale(l.c1, p.x), F2::scale(l.c2, p.y));
    }
  }
  return F12::conj(f);
}

}  // namespace
}  // namespace b200zk
