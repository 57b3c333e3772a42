// bn_pairing.cuh -- the stages of the BN254 ate pairing: the affine line function, the Miller loop and the final
// exponentiation, and the EIP-196/197 point decoding.  pairing.cu builds the ecPairing kernels on them, groth16_verify.cu
// the batched Groth16 check; tests/csrc/pairing_conformance.cu runs each stage alone.  See pairing.cu for the algorithm.
// Internal linkage (anonymous namespace, __constant__ tables): the build has no -rdc, so each translation unit that
// includes this header holds its own copy.
#pragma once
#include "common.cuh"
#include "curve.cuh"
#include "tower.cuh"

namespace b200zk {
namespace {

__constant__ uint32_t kAteT[4] = {0xe87cfd46u, 0xf83e9682u, 0xeeb859fbu, 0x6f4d8248u};  // 6x^2, x = 4965661367192848881
static constexpr int kAteBits = 127;
__constant__ uint32_t kFinalExp[40] = {  // (p^6 + 1) / r, 1268 bits
    0x36e3f812u, 0x5250a540u, 0x96789051u, 0xa5635f15u, 0x4d5bd1d4u, 0xd1138bf5u, 0xbe36c7a2u, 0xa8ce2533u, 0x84e09bf6u, 0x94f69f6bu,
    0x50ef3644u, 0x42ad1f5eu, 0x48c3454cu, 0x0fcc420eu, 0xecc9952cu, 0x758e4408u, 0x87c6042cu, 0xc901bf18u, 0xb14bb3b5u, 0xa733cd65u,
    0xcf51b0d8u, 0xdf6d76bdu, 0x82eb59e1u, 0xca64c0fdu, 0xe39276a1u, 0x1d2e5726u, 0xa391cae9u, 0xc2d1ea74u, 0xc82d647eu, 0x07409206u,
    0xa5afdd17u, 0x051c6d1au, 0x19667af5u, 0xb37f6019u, 0x5084015bu, 0x150e578cu, 0xc23998e4u, 0xfbdea556u, 0xc52f5b83u, 0x000fd14cu};
static constexpr int kFinalExpBits = 1268;

typedef Fp12<Fq2> Fq12;
typedef TowerF2<Fq2> M2;  // the non-inlined Fq2 product and inverse

B2_D Fq2 f2_scale(const Fq2& a, const Fq& k) { return {Fq::mul(a.c0, k), Fq::mul(a.c1, k)}; }

// l(P) = yP - (lam xP) w + (lam xT - yT) w^3, w^3 = v w
B2_D Fq12 line_at(const Fq2& lam, const Fq2& xt, const Fq2& yt, const Affine<Fq>& p) {
  Fq12 l;
  l.c0 = {{p.y, Fq::zero()}, Fq2::zero(), Fq2::zero()};
  l.c1 = {Fq2::neg(f2_scale(lam, p.x)), Fq2::sub(M2::mul(lam, xt), yt), Fq2::zero()};
  return l;
}

// f_{T,Q}(P); neither point is the identity, Q has order r (so no step meets an exceptional case: T < r)
__device__ __noinline__ Fq12 miller_ate(const Affine<Fq2>& q, const Affine<Fq>& p) {
  Fq12 f = Fq12::one();
  Fq2 rx = q.x, ry = q.y;
  for (int i = kAteBits - 2; i >= 0; --i) {
    Fq2 xx = M2::mul(rx, rx);
    Fq2 lam = M2::mul(Fq2::add(Fq2::dbl(xx), xx), M2::inv(Fq2::dbl(ry)));
    f = Fq12::mul(Fq12::mul(f, f), line_at(lam, rx, ry, p));
    Fq2 nx = Fq2::sub(Fq2::sub(M2::mul(lam, lam), rx), rx);
    ry = Fq2::sub(M2::mul(lam, Fq2::sub(rx, nx)), ry);
    rx = nx;
    if ((kAteT[i >> 5] >> (i & 31)) & 1) {
      lam = M2::mul(Fq2::sub(ry, q.y), M2::inv(Fq2::sub(rx, q.x)));
      f = Fq12::mul(f, line_at(lam, rx, ry, p));
      nx = Fq2::sub(Fq2::sub(M2::mul(lam, lam), rx), q.x);
      ry = Fq2::sub(M2::mul(lam, Fq2::sub(rx, nx)), ry);
      rx = nx;
    }
  }
  return f;
}

// the Miller value of one pair of decoded points: 1 when either is the identity (the pair contributes nothing)
B2_D Fq12 miller_pair(const Affine<Fq>& p, const Affine<Fq2>& q) {
  return (p.is_inf() || q.is_inf()) ? Fq12::one() : miller_ate(q, p);
}

__device__ __noinline__ Fq12 final_exponentiate(const Fq12& f) {
  Fq12 b = Fq12::mul(Fq12::conj(f), Fq12::inv(f));  // f^(p^6 - 1)
  Fq12 acc = Fq12::one();
  for (int i = kFinalExpBits - 1; i >= 0; --i) {
    acc = Fq12::mul(acc, acc);
    if ((kFinalExp[i >> 5] >> (i & 31)) & 1) acc = Fq12::mul(acc, b);
  }
  return acc;
}

// ---- decoding with the precompile's error order: field range first, then the curve ---------------------------
// a 32-byte big-endian value as limbs of F (not reduced); *in_range = value < the modulus
template <class F> B2_D F load_be(const uint8_t* in, bool* in_range) {
  F v;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint8_t* b = in + 4 * (7 - k);
    v.v[k] = ((uint32_t)b[0] << 24) | ((uint32_t)b[1] << 16) | ((uint32_t)b[2] << 8) | (uint32_t)b[3];
  }
  F m = F::modulus(), t;
  *in_range = detail::sub8(t.v, v.v, m.v) != 0;
  return v;
}
// 0 ok, 2 coordinate >= p, 3 not on the curve
B2_D uint32_t decode_g1(const uint8_t* be, Affine<Fq>* out) {
  bool okx, oky;
  Fq x = load_be<Fq>(be, &okx), y = load_be<Fq>(be + 32, &oky);
  if (!(okx && oky)) return B200ZK_ERR_NOT_IN_FIELD;
  *out = {Fq::to_mont(x), Fq::to_mont(y)};
  return affine_on_curve(*out) ? 0u : (uint32_t)B200ZK_ERR_NOT_ON_CURVE;
}
B2_D uint32_t decode_g2(const uint8_t* be, Affine<Fq2>* out) {
  bool ok[4];
  Fq xi = load_be<Fq>(be, &ok[0]), xr = load_be<Fq>(be + 32, &ok[1]), yi = load_be<Fq>(be + 64, &ok[2]), yr = load_be<Fq>(be + 96, &ok[3]);
  if (!(ok[0] && ok[1] && ok[2] && ok[3])) return B200ZK_ERR_NOT_IN_FIELD;
  *out = {{Fq::to_mont(xr), Fq::to_mont(xi)}, {Fq::to_mont(yr), Fq::to_mont(yi)}};
  return affine_on_curve(*out) ? 0u : (uint32_t)B200ZK_ERR_NOT_ON_CURVE;
}

}  // namespace
}  // namespace b200zk
