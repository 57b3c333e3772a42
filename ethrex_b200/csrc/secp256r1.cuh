// secp256r1.cuh -- P-256 (secp256r1, NIST P-256) ECDSA verification for one item per thread: the P256VERIFY precompile
// of EIP-7951 (address 0x100).  The base field p = 2^256 - 2^224 + 2^192 + 2^96 - 1 and the scalar field n are both
// Montgomery fields over 32-bit limbs; the curve y^2 = x^3 - 3x + b runs through curve.cuh's templates with CurveA = -3,
// and u1 G + u2 Q through the same ladder and G table shape as secp256k1 (secp_lincomb, secp256k1.cuh).  Every function
// is __host__ __device__ and portable C++ (no inline PTX), so the tests compile this header for the host with nvcc and
// compare it with a Python oracle without a device; the kernel runs the same code.
//
// Semantics are those of the reference's Crypto::secp256r1_verify (the p256 crate's VerifyingKey::verify_prehash) and of
// EIP-7951; see p256_verify below for the rules in order.
#pragma once
#include "secp256k1.cuh"  // the 256-bit limb helpers (secp::) and the ECDSA ladder (secp_wnaf, secp_lincomb, ecdsa_g_multiple)

namespace b200zk {

namespace p256 {
// little-endian 32-bit limbs
B2_HD constexpr uint32_t P(int i) {  // p = 2^256 - 2^224 + 2^192 + 2^96 - 1
  constexpr uint32_t m[8] = {0xffffffffu, 0xffffffffu, 0xffffffffu, 0x00000000u, 0x00000000u, 0x00000000u, 0x00000001u, 0xffffffffu};
  return m[i];
}
B2_HD constexpr uint32_t N(int i) {  // the group order n (the cofactor is 1)
  constexpr uint32_t m[8] = {0xfc632551u, 0xf3b9cac2u, 0xa7179e84u, 0xbce6faadu, 0xffffffffu, 0xffffffffu, 0x00000000u, 0xffffffffu};
  return m[i];
}
B2_HD constexpr uint32_t P_MINUS_N(int i) {  // p - n < 2^127: x(R') = r + n is possible only for r < p - n
  constexpr uint32_t m[8] = {0x039cdaaeu, 0x0c46353du, 0x58e8617bu, 0x43190553u, 0u, 0u, 0u, 0u};
  return m[i];
}
B2_HD constexpr uint32_t B(int i) {  // the curve's b, canonical
  constexpr uint32_t m[8] = {0x27d2604bu, 0x3bce3c3eu, 0xcc53b0f6u, 0x651d06b0u, 0x769886bcu, 0xb3ebbd55u, 0xaa3a93e7u, 0x5ac635d8u};
  return m[i];
}
B2_HD constexpr uint32_t GX(int i) {
  constexpr uint32_t m[8] = {0xd898c296u, 0xf4a13945u, 0x2deb33a0u, 0x77037d81u, 0x63a440f2u, 0xf8bce6e5u, 0xe12c4247u, 0x6b17d1f2u};
  return m[i];
}
B2_HD constexpr uint32_t GY(int i) {
  constexpr uint32_t m[8] = {0x37bf51f5u, 0xcbb64068u, 0x6b315eceu, 0x2bce3357u, 0x7c0f9e16u, 0x8ee7eb4au, 0xfe1a7f9bu, 0x4fe342e2u};
  return m[i];
}
// the two moduli for P256Mont: limbs, 2^256 mod m (Montgomery one), 2^512 mod m (to_mont) and -m^-1 mod 2^32
struct FpMod {
  static B2_HD constexpr uint32_t m(int i) { return P(i); }
  static B2_HD constexpr uint32_t r1(int i) {
    constexpr uint32_t v[8] = {0x00000001u, 0x00000000u, 0x00000000u, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xfffffffeu, 0x00000000u};
    return v[i];
  }
  static B2_HD constexpr uint32_t r2(int i) {
    constexpr uint32_t v[8] = {0x00000003u, 0x00000000u, 0xffffffffu, 0xfffffffbu, 0xfffffffeu, 0xffffffffu, 0xfffffffdu, 0x00000004u};
    return v[i];
  }
  static constexpr uint32_t inv = 1;  // p = -1 (mod 2^32), so every CIOS round's multiplier is t[0] itself
};
struct FnMod {
  static B2_HD constexpr uint32_t m(int i) { return N(i); }
  static B2_HD constexpr uint32_t r1(int i) {
    constexpr uint32_t v[8] = {0x039cdaafu, 0x0c46353du, 0x58e8617bu, 0x43190552u, 0x00000000u, 0x00000000u, 0xffffffffu, 0x00000000u};
    return v[i];
  }
  static B2_HD constexpr uint32_t r2(int i) {
    constexpr uint32_t v[8] = {0xbe79eea2u, 0x83244c95u, 0x49bd6fa6u, 0x4699799cu, 0x2b6bec59u, 0x2845b239u, 0xf3d95620u, 0x66e12d94u};
    return v[i];
  }
  static constexpr uint32_t inv = 0xee00bc4fu;
};
}  // namespace p256

// ---- P256Fp, P256Fn: Montgomery (R = 2^256) over a modulus m that fills all 256 bits -------------------------------------
// Values are canonical Montgomery residues 0 <= v < m.  m > 2^255, so there is no headroom: add keeps the carry out of
// limb 7, and the CIOS product keeps its running total in nine limbs plus a carry.
template <class M> struct P256Mont {
  uint32_t v[8];

  static B2_HD P256Mont zero() { P256Mont r; for (int i = 0; i < 8; ++i) r.v[i] = 0; return r; }
  static B2_HD P256Mont one() { P256Mont r; secp::load_const(r.v, M::r1); return r; }
  static B2_HD P256Mont modulus() { P256Mont r; secp::load_const(r.v, M::m); return r; }
  B2_HD bool is_zero() const {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) o |= v[i];
    return o == 0;
  }
  B2_HD bool operator==(const P256Mont& b) const {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) o |= v[i] ^ b.v[i];
    return o == 0;
  }
  B2_HD bool operator!=(const P256Mont& b) const { return !(*this == b); }

  // a, b < m: the sum is < 2m < 2^257.  With the carry c, s + c 2^256 >= m exactly when c is set or s - m does not borrow.
  static B2_HD P256Mont add(const P256Mont& a, const P256Mont& b) {
    P256Mont s, t, m = modulus();
    const uint32_t c = secp::add256(s.v, a.v, b.v);
    const uint32_t bo = secp::sub256(t.v, s.v, m.v);
    return (c | !bo) ? t : s;
  }
  // a, b < m: on a borrow a - b + 2^256 + m wraps to a - b + m < m
  static B2_HD P256Mont sub(const P256Mont& a, const P256Mont& b) {
    P256Mont d, m = modulus();
    if (secp::sub256(d.v, a.v, b.v)) secp::add256(d.v, d.v, m.v);
    return d;
  }
  static B2_HD P256Mont dbl(const P256Mont& a) { return add(a, a); }
  static B2_HD P256Mont neg(const P256Mont& a) { return a.is_zero() ? a : sub(zero(), a); }

  // a, b < m -> a b / 2^256 mod m (CIOS).  Round i adds a b_i (< m 2^32) and q m (< m 2^32) to t < 2m and divides by
  // 2^32, so t stays < (2m + 2 m (2^32 - 1)) / 2^32 = 2m < 2^257: nine limbs t[0..8], with t[9] the carry of one round's
  // sum before the division.  One conditional subtraction (taken also when t[8] is set) canonicalises the result.
  static B2_HD P256Mont mul(const P256Mont& a, const P256Mont& b) {
    uint32_t t[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 8; ++i) {
      uint64_t c = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { c += (uint64_t)t[j] + (uint64_t)a.v[j] * b.v[i]; t[j] = (uint32_t)c; c >>= 32; }
      c += t[8]; t[8] = (uint32_t)c; t[9] = (uint32_t)(c >> 32);
      const uint32_t q = t[0] * M::inv;
      c = ((uint64_t)t[0] + (uint64_t)q * M::m(0)) >> 32;
#pragma unroll
      for (int j = 1; j < 8; ++j) { c += (uint64_t)t[j] + (uint64_t)q * M::m(j); t[j - 1] = (uint32_t)c; c >>= 32; }
      c += t[8]; t[7] = (uint32_t)c; c >>= 32;
      t[8] = t[9] + (uint32_t)c;
    }
    P256Mont r, s, m = modulus();
#pragma unroll
    for (int i = 0; i < 8; ++i) r.v[i] = t[i];
    const uint32_t bo = secp::sub256(s.v, r.v, m.v);
    return (t[8] | !bo) ? s : r;
  }
  static B2_HD P256Mont sqr(const P256Mont& a) { return mul(a, a); }
  static B2_HD P256Mont mul2_sub(const P256Mont& a, const P256Mont& b, const P256Mont& c, const P256Mont& d) { return sub(mul(a, b), mul(c, d)); }
  static B2_HD P256Mont to_mont(const P256Mont& a) { P256Mont r2; secp::load_const(r2.v, M::r2); return mul(a, r2); }  // a < m
  static B2_HD P256Mont from_mont(const P256Mont& a) { P256Mont o = zero(); o.v[0] = 1; return mul(a, o); }
  // a^e, e = 256-bit little-endian limbs (square-and-multiply, MSB first), Montgomery in and out
  static B2_HD P256Mont pow(const P256Mont& a, const uint32_t* e) {
    P256Mont acc = one();
    for (int i = 255; i >= 0; --i) {
      acc = sqr(acc);
      if ((e[i >> 5] >> (i & 31)) & 1) acc = mul(acc, a);
    }
    return acc;
  }
  static B2_HD P256Mont inv(const P256Mont& a) {  // Fermat: a^(m-2); inv(0) = 0
    uint32_t e[8];
    secp::load_const(e, M::m);
    e[0] -= 2;  // p ends in ...ffffffff, n in ...fc632551: no borrow
    return pow(a, e);
  }
};
using P256Fp = P256Mont<p256::FpMod>;
using P256Fn = P256Mont<p256::FnMod>;

template <> struct CurveA<P256Fp> { static constexpr int a = -3; };
template <> struct CurveB<P256Fp> {
  static B2_HD P256Fp b() { P256Fp s; secp::load_const(s.v, p256::B); return P256Fp::to_mont(s); }
};

// ---- verification ---------------------------------------------------------------------------------------------------------
// an entry of the affine table (Montgomery form) the G term reads: table[d - 1] = d G, d = 1 .. kSecpGTable
B2_HD Affine<P256Fp> p256_g_multiple(uint32_t d) {
  Affine<P256Fp> g;
  secp::load_const(g.x.v, p256::GX);
  secp::load_const(g.y.v, p256::GY);
  g.x = P256Fp::to_mont(g.x);
  g.y = P256Fp::to_mont(g.y);
  return ecdsa_g_multiple(g, d);
}

// One P256VERIFY item: in = h | r | s | qx | qy, five 32-byte big-endian words (160 bytes).  True when the signature
// verifies.  The rules in order, the first failure decides (false):
//   1. r or s outside [1, n - 1]
//   2. qx >= p or qy >= p (never reduced)
//   3. (qx, qy) not on y^2 = x^3 - 3x + b; (0, 0) is not a curve point.  The cofactor is 1: no subgroup check.
//   4. z = h mod n (h as a 256-bit integer); R' = (z / s) G + (r / s) Q; R' = O
//   5. x(R') mod n != r.  x(R') < p < 2n, so x(R') mod n = r means x(R') = r, or x(R') = r + n when r + n < p.
// High s is accepted: (r, s) and (r, n - s) both verify.
B2_HD bool p256_verify(const uint8_t* in, const Affine<P256Fp>* gtab) {
  uint32_t h[8], r[8], s[8], k[8];
  P256Fp qx, qy;
  secp::load_be256(h, in);
  secp::load_be256(r, in + 32);
  secp::load_be256(s, in + 64);
  secp::load_be256(qx.v, in + 96);
  secp::load_be256(qy.v, in + 128);
  secp::load_const(k, p256::N);
  uint32_t rz = 0, sz = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) { rz |= r[i]; sz |= s[i]; }
  if (!rz || !sz || !secp::less256(r, k) || !secp::less256(s, k)) return false;
  const P256Fp p = P256Fp::modulus();
  if (!secp::less256(qx.v, p.v) || !secp::less256(qy.v, p.v)) return false;
  Affine<P256Fp> Q;
  Q.x = P256Fp::to_mont(qx);
  Q.y = P256Fp::to_mont(qy);
  if (Q.is_inf() || !affine_on_curve(Q)) return false;  // affine_on_curve takes (0, 0) for the identity
  uint32_t zr[8];
  if (!secp::sub256(zr, h, k)) {  // h < 2^256 < 2n: one subtraction reduces it
#pragma unroll
    for (int i = 0; i < 8; ++i) h[i] = zr[i];
  }
  // w = s^-1 in Montgomery form (s^-1 2^256); the Montgomery product of a canonical value with w is canonical value / s
  P256Fn sn, zn, rn;
#pragma unroll
  for (int i = 0; i < 8; ++i) { sn.v[i] = s[i]; zn.v[i] = h[i]; rn.v[i] = r[i]; }
  const P256Fn w = P256Fn::inv(P256Fn::to_mont(sn));
  const P256Fn u1 = P256Fn::mul(zn, w), u2 = P256Fn::mul(rn, w);
  const XYZZ<P256Fp> R = secp_lincomb(u1.v, u2.v, Q, gtab);
  if (R.is_inf()) return false;
  // x(R') = X / ZZ: compare r ZZ with X, and (r + n) ZZ when r + n < p, without inverting ZZ
  P256Fp xr;
#pragma unroll
  for (int i = 0; i < 8; ++i) xr.v[i] = r[i];  // r < n < p
  if (P256Fp::mul(P256Fp::to_mont(xr), R.zz) == R.x) return true;
  secp::load_const(zr, p256::P_MINUS_N);
  if (!secp::less256(r, zr)) return false;
  secp::add256(xr.v, r, k);  // r + n < p
  return P256Fp::mul(P256Fp::to_mont(xr), R.zz) == R.x;
}

}  // namespace b200zk
