// tower.cuh -- the degree-12 tower both pairings compute in, over a quadratic extension F2 = Fp[u]/(u^2 + 1):
//   Fp6 = F2[v]/(v^3 - xi), Fp12 = Fp6[w]/(w^2 - v),  xi = 9 + u for BN254 (Fq2), 1 + u for BLS12-381 (Fp2_381),
// and the pairing-check kernel both end in.  F2 provides zero, one, add, sub, neg, mul, sqr, inv, is_zero, == and mul_xi
// (the product by xi).  Bit-exact against the schoolbook model of tests/field_conformance_ref.py.
//
// The tower is latency-bound single-thread code and compiles slowly, so the heavy routines are __noinline__: the build
// has no -rdc, so each translation unit keeps one device copy of each.  For the same reason every kernel reaches the F2
// product and inverse through one non-inlined function each: TowerF2<F2>::mul and inv.
#pragma once
#include "common.cuh"

namespace b200zk {

// Fp2_381's mul and inv are non-inlined themselves
template <class F2> struct TowerF2 {
  static B2_D F2 mul(const F2& a, const F2& b) { return F2::mul(a, b); }
  static B2_D F2 sqr(const F2& a) { return F2::sqr(a); }
  static B2_D F2 inv(const F2& a) { return F2::inv(a); }
};
// Fq2's are inlined, because they are the G2 MSM's hot path: the tower calls them through these wrappers, and squares
// with the non-inlined product rather than another inlined copy of Fq2::sqr
template <> struct TowerF2<Fq2> {
  static __device__ __noinline__ Fq2 mul(const Fq2& a, const Fq2& b) { return Fq2::mul(a, b); }
  static B2_D Fq2 sqr(const Fq2& a) { return mul(a, a); }
  static __device__ __noinline__ Fq2 inv(const Fq2& a) { return Fq2::inv(a); }
};

template <class F2> struct Fp6 {
  F2 c0, c1, c2;
  typedef TowerF2<F2> M;
  static B2_D Fp6 zero() { return {F2::zero(), F2::zero(), F2::zero()}; }
  static B2_D Fp6 one() { return {F2::one(), F2::zero(), F2::zero()}; }
  static B2_D Fp6 add(const Fp6& a, const Fp6& b) { return {F2::add(a.c0, b.c0), F2::add(a.c1, b.c1), F2::add(a.c2, b.c2)}; }
  static B2_D Fp6 sub(const Fp6& a, const Fp6& b) { return {F2::sub(a.c0, b.c0), F2::sub(a.c1, b.c1), F2::sub(a.c2, b.c2)}; }
  static B2_D Fp6 neg(const Fp6& a) { return {F2::neg(a.c0), F2::neg(a.c1), F2::neg(a.c2)}; }
  static B2_D Fp6 mul_v(const Fp6& a) { return {F2::mul_xi(a.c2), a.c0, a.c1}; }
  static __device__ __noinline__ Fp6 mul(const Fp6& a, const Fp6& b) {  // Karatsuba over F2: six products
    const F2 t0 = M::mul(a.c0, b.c0), t1 = M::mul(a.c1, b.c1), t2 = M::mul(a.c2, b.c2);
    Fp6 r;
    r.c0 = F2::add(t0, F2::mul_xi(F2::sub(F2::sub(M::mul(F2::add(a.c1, a.c2), F2::add(b.c1, b.c2)), t1), t2)));
    r.c1 = F2::add(F2::sub(F2::sub(M::mul(F2::add(a.c0, a.c1), F2::add(b.c0, b.c1)), t0), t1), F2::mul_xi(t2));
    r.c2 = F2::add(F2::sub(F2::sub(M::mul(F2::add(a.c0, a.c2), F2::add(b.c0, b.c2)), t0), t2), t1);
    return r;
  }
  // a (b0 + b1 v): the shape of a BLS12-381 line
  static __device__ __noinline__ Fp6 mul_01(const Fp6& a, const F2& b0, const F2& b1) {
    return {F2::add(M::mul(a.c0, b0), F2::mul_xi(M::mul(a.c2, b1))), F2::add(M::mul(a.c0, b1), M::mul(a.c1, b0)),
            F2::add(M::mul(a.c1, b1), M::mul(a.c2, b0))};
  }
  static B2_D Fp6 mul_1(const Fp6& a, const F2& b1) { return {F2::mul_xi(M::mul(a.c2, b1)), M::mul(a.c0, b1), M::mul(a.c1, b1)}; }
  static __device__ __noinline__ Fp6 inv(const Fp6& a) {  // inv(0) = 0
    const F2 A = F2::sub(M::sqr(a.c0), F2::mul_xi(M::mul(a.c1, a.c2)));
    const F2 B = F2::sub(F2::mul_xi(M::sqr(a.c2)), M::mul(a.c0, a.c1));
    const F2 C = F2::sub(M::sqr(a.c1), M::mul(a.c0, a.c2));
    const F2 Fi = M::inv(F2::add(M::mul(a.c0, A), F2::mul_xi(F2::add(M::mul(a.c2, B), M::mul(a.c1, C)))));
    return {M::mul(A, Fi), M::mul(B, Fi), M::mul(C, Fi)};
  }
};

template <class F2> struct Fp12 {
  typedef Fp6<F2> F6;
  F6 c0, c1;
  static B2_D Fp12 one() { return {F6::one(), F6::zero()}; }
  static B2_D bool is_one(const Fp12& a) {
    return a.c0.c0 == F2::one() && a.c0.c1.is_zero() && a.c0.c2.is_zero() && a.c1.c0.is_zero() && a.c1.c1.is_zero() && a.c1.c2.is_zero();
  }
  static B2_D Fp12 conj(const Fp12& a) { return {a.c0, F6::neg(a.c1)}; }
  // Karatsuba over Fp6: three products.  c1 first: c0 is not live across the third product, which keeps spills down
  static __device__ __noinline__ Fp12 mul(const Fp12& a, const Fp12& b) {
    const F6 t0 = F6::mul(a.c0, b.c0), t1 = F6::mul(a.c1, b.c1);
    Fp12 r;
    r.c1 = F6::sub(F6::sub(F6::mul(F6::add(a.c0, a.c1), F6::add(b.c0, b.c1)), t0), t1);
    r.c0 = F6::add(t0, F6::mul_v(t1));
    return r;
  }
  static __device__ __noinline__ Fp12 sqr(const Fp12& a) {  // complex squaring: two Fp6 products
    const F6 ab = F6::mul(a.c0, a.c1);
    const F6 c0 = F6::sub(F6::sub(F6::mul(F6::add(a.c0, a.c1), F6::add(a.c0, F6::mul_v(a.c1))), ab), F6::mul_v(ab));
    return {c0, F6::add(ab, ab)};
  }
  // f (c0 + c1 v + c4 v w): aa = f.c0 (c0 + c1 v), bb = f.c1 (c4 v), then Karatsuba over Fp6
  static __device__ __noinline__ Fp12 mul_014(const Fp12& f, const F2& c0, const F2& c1, const F2& c4) {
    const F6 aa = F6::mul_01(f.c0, c0, c1), bb = F6::mul_1(f.c1, c4);
    const F6 t = F6::mul_01(F6::add(f.c0, f.c1), c0, F2::add(c1, c4));
    return {F6::add(aa, F6::mul_v(bb)), F6::sub(F6::sub(t, aa), bb)};
  }
  static __device__ __noinline__ Fp12 inv(const Fp12& a) {  // inv(0) = 0
    const F6 t = F6::inv(F6::sub(F6::mul(a.c0, a.c0), F6::mul_v(F6::mul(a.c1, a.c1))));
    return {F6::mul(a.c0, t), F6::neg(F6::mul(a.c1, t))};
  }
};

constexpr uint8_t kTrivial = 0x80;  // pair status bit: a side is the identity, the pair contributes 1 (BLS12-381 only)

// One thread per check: the product of its pairs' Miller values f[lo, hi), one final exponentiation, compared with 1.  A
// range error anywhere in the check outranks a curve error (every point is range-checked before any curve check).  A check
// without pairs is true and skips the exponentiation.
template <class F12, F12 (*FinalExp)(const F12&)>
__global__ void __launch_bounds__(32) pairing_check(const F12* f, const uint8_t* pst, const uint32_t* offsets, size_t count, uint8_t* result, uint8_t* status) {
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
    F12 acc = F12::one();
    for (uint32_t k = lo; k < hi; ++k) acc = F12::mul(acc, f[k]);
    ok = (hi == lo) ? 1u : (F12::is_one(FinalExp(acc)) ? 1u : 0u);
  }
  result[i] = (uint8_t)ok;
  status[i] = (uint8_t)s;
}

}  // namespace b200zk
