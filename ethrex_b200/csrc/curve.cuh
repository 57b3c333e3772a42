// curve.cuh -- BN254 G1 (over Fq) and G2 (over Fq2) group law for sm_90a, y^2 = x^3 + b, a = 0.
//
// Affine points are the HBM-resident base format: (x, y) in Montgomery form, (0,0) = identity (the
// EIP-196/197 convention of /root/reference/crates/common/crypto/provider.rs:201-330).  Accumulators use
// extended Jacobian "XYZZ" coordinates (x = X/ZZ, y = Y/ZZZ, ZZ^3 = ZZZ^2; ZZ = 0 = identity): the mixed
// addition costs 8M+2S and needs no inversion, which is what the bucket-accumulation kernel is made of.
// Formulas: EFD shortw/xyzz madd-2008-s, add-2008-s, dbl-2008-s-1, mdbl-2008-s-1 (a = 0; CurveA below adds a = -3
// for P-256, which only the doublings and the curve equation see).  The affine
// result of an MSM is independent of the coordinate system, so bit-exactness against the reference's
// Jacobian arithmetic (ark-ec 0.5.0 short_weierstrass::Projective) only depends on the final normalisation.
// The templates are __host__ __device__: a field type whose operations are too (secp256k1.cuh) runs them on the host,
// which is how its tests check them without a device; the device-only fields only ever instantiate them in kernels.
#pragma once
#include "field.cuh"

namespace b200zk {

template <class F> struct Affine {
  F x, y;
  B2_HD bool is_inf() const { return x.is_zero() && y.is_zero(); }
};

template <class F> struct XYZZ {
  F x, y, zz, zzz;
  static B2_HD XYZZ identity() { return {F::zero(), F::zero(), F::zero(), F::zero()}; }
  B2_HD bool is_inf() const { return zz.is_zero(); }
};

template <class F> B2_HD XYZZ<F> xyzz_from_affine(const Affine<F>& p) {
  if (p.is_inf()) return XYZZ<F>::identity();
  return {p.x, p.y, F::one(), F::one()};
}

// the a coefficient of y^2 = x^3 + a x + b: 0 unless a curve specialises it.  The doublings and affine_on_curve support
// a = 0 and a = -3 (P-256, secp256r1.cuh); for a = 0 they compile to exactly the a-free formulas.
template <class F> struct CurveA { static constexpr int a = 0; };

// 2*(x1, y1) for an affine point (mdbl-2008-s-1); M = 3 x^2 + a
template <class F> B2_HD XYZZ<F> xyzz_mdbl(const F& x1, const F& y1) {
  static_assert(CurveA<F>::a == 0 || CurveA<F>::a == -3, "curve.cuh doubles only for a = 0 or a = -3");
  F U = F::dbl(y1), V = F::sqr(U), W = F::mul(U, V), S = F::mul(x1, V);
  F M;
  if constexpr (CurveA<F>::a == -3) {  // 3 (x - 1)(x + 1)
    F t = F::mul(F::sub(x1, F::one()), F::add(x1, F::one()));
    M = F::add(F::dbl(t), t);
  } else {
    F xx = F::sqr(x1);
    M = F::add(F::dbl(xx), xx);
  }
  XYZZ<F> r;
  r.x = F::sub(F::sqr(M), F::dbl(S));
  r.y = F::mul2_sub(M, F::sub(S, r.x), W, y1);
  r.zz = V; r.zzz = W;
  return r;
}

// 2*P (dbl-2008-s-1); M = 3 X^2 + a ZZ^2
template <class F> B2_HD XYZZ<F> xyzz_dbl(const XYZZ<F>& p) {
  static_assert(CurveA<F>::a == 0 || CurveA<F>::a == -3, "curve.cuh doubles only for a = 0 or a = -3");
  if (p.is_inf()) return p;
  F U = F::dbl(p.y), V = F::sqr(U), W = F::mul(U, V), S = F::mul(p.x, V);
  F M;
  if constexpr (CurveA<F>::a == -3) {  // 3 (X - ZZ)(X + ZZ)
    F t = F::mul(F::sub(p.x, p.zz), F::add(p.x, p.zz));
    M = F::add(F::dbl(t), t);
  } else {
    F xx = F::sqr(p.x);
    M = F::add(F::dbl(xx), xx);
  }
  XYZZ<F> r;
  r.x = F::sub(F::sqr(M), F::dbl(S));
  r.y = F::mul2_sub(M, F::sub(S, r.x), W, p.y);
  r.zz = F::mul(V, p.zz); r.zzz = F::mul(W, p.zzz);
  return r;
}

// acc += (x2, y2)  (madd-2008-s; identity, doubling and cancellation handled)
template <class F> B2_HD void xyzz_add_mixed(XYZZ<F>& acc, const F& x2, const F& y2) {
  if (x2.is_zero() && y2.is_zero()) return;
  if (acc.is_inf()) { acc.x = x2; acc.y = y2; acc.zz = F::one(); acc.zzz = F::one(); return; }
  F U2 = F::mul(x2, acc.zz), S2 = F::mul(y2, acc.zzz);
  F P = F::sub(U2, acc.x), R = F::sub(S2, acc.y);
  if (P.is_zero()) {
    if (R.is_zero()) acc = xyzz_mdbl(x2, y2);
    else acc = XYZZ<F>::identity();
    return;
  }
  F PP = F::sqr(P), PPP = F::mul(P, PP), Q = F::mul(acc.x, PP);
  F x3 = F::sub(F::sub(F::sqr(R), PPP), F::dbl(Q));
  acc.y = F::mul2_sub(R, F::sub(Q, x3), acc.y, PPP);
  acc.x = x3;
  acc.zz = F::mul(acc.zz, PP);
  acc.zzz = F::mul(acc.zzz, PPP);
}

// acc += q  (add-2008-s with the exceptional cases)
template <class F> B2_HD void xyzz_add(XYZZ<F>& acc, const XYZZ<F>& q) {
  if (q.is_inf()) return;
  if (acc.is_inf()) { acc = q; return; }
  F U1 = F::mul(acc.x, q.zz), U2 = F::mul(q.x, acc.zz);
  F S1 = F::mul(acc.y, q.zzz), S2 = F::mul(q.y, acc.zzz);
  F P = F::sub(U2, U1), R = F::sub(S2, S1);
  if (P.is_zero()) {
    if (R.is_zero()) acc = xyzz_dbl(acc);
    else acc = XYZZ<F>::identity();
    return;
  }
  F PP = F::sqr(P), PPP = F::mul(P, PP), Q = F::mul(U1, PP);
  F x3 = F::sub(F::sub(F::sqr(R), PPP), F::dbl(Q));
  acc.y = F::mul2_sub(R, F::sub(Q, x3), S1, PPP);
  acc.x = x3;
  acc.zz = F::mul(F::mul(acc.zz, q.zz), PP);
  acc.zzz = F::mul(F::mul(acc.zzz, q.zzz), PPP);
}

template <class F> B2_HD Affine<F> xyzz_to_affine(const XYZZ<F>& p) {
  if (p.is_inf()) return {F::zero(), F::zero()};
  F t = F::inv(F::mul(p.zz, p.zzz));
  F zz_inv = F::mul(t, p.zzz), zzz_inv = F::mul(t, p.zz);
  return {F::mul(p.x, zz_inv), F::mul(p.y, zzz_inv)};
}

// k * P, k = 256-bit little-endian limbs (double-and-add, MSB first).  Setup / utility use only.
template <class F> B2_HD XYZZ<F> xyzz_scalar_mul(const uint32_t* k, const Affine<F>& p) {
  XYZZ<F> acc = XYZZ<F>::identity();
  for (int i = 255; i >= 0; --i) {
    acc = xyzz_dbl(acc);
    if ((k[i >> 5] >> (i & 31)) & 1) xyzz_add_mixed(acc, p.x, p.y);
  }
  return acc;
}

// the subgroup check r P = O (no endomorphism shortcuts), Order(j) = limb j of the group order r (8 little-endian limbs):
// FrCfg::mod for BN254, bls_r_limb for BLS12-381.  Non-inlined: one copy per translation unit and group.
template <uint32_t (*Order)(int), class F> __device__ __noinline__ bool in_subgroup(const Affine<F>& p) {
  uint32_t k[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) k[j] = Order(j);
  return xyzz_scalar_mul<F>(k, p).is_inf();
}

// curve constants in Montgomery form
template <class F> struct CurveB;
template <> struct CurveB<Fq> {
  static B2_D Fq b() {  // 3 * R mod p
    Fq three = Fq::zero(); three.v[0] = 3; return Fq::to_mont(three);
  }
};
template <> struct CurveB<Fq2> {
  static B2_D Fq2 b() {  // 3/(9+u): canonical values cross-checked in oracle/pyref.py (B_G2)
    const uint32_t re[8] = {0x24a138e5u, 0x3267e6dcu, 0x59dbefa3u, 0xb5b4c5e5u, 0x1be06ac3u, 0x81be1899u, 0xceb8aaaeu, 0x2b149d40u};
    const uint32_t im[8] = {0x85c315d2u, 0xe4a2bd06u, 0xe52d1852u, 0xa74fa084u, 0xeed8fdf4u, 0xcd2cafadu, 0x3af0fed4u, 0x009713b0u};
    Fq a, c;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a.v[i] = re[i]; c.v[i] = im[i]; }
    return {Fq::to_mont(a), Fq::to_mont(c)};
  }
};
template <class F> B2_HD bool affine_on_curve(const Affine<F>& p) {
  static_assert(CurveA<F>::a == 0 || CurveA<F>::a == -3, "curve.cuh checks the curve equation only for a = 0 or a = -3");
  if (p.is_inf()) return true;
  F lhs = F::sqr(p.y), rhs;
  if constexpr (CurveA<F>::a == -3) rhs = F::add(F::mul(F::sub(F::sqr(p.x), F::add(F::dbl(F::one()), F::one())), p.x), CurveB<F>::b());  // (x^2 - 3) x + b
  else rhs = F::add(F::mul(F::sqr(p.x), p.x), CurveB<F>::b());
  return lhs == rhs;
}

}  // namespace b200zk
