// bls12.cuh -- BLS12-381 pieces shared by bls381.cu (commitments, proofs), bls_pairing.cu (the pairing, KZG verification)
// and bls_ops.cu (EIP-2537 addition and MSM): big-endian byte loaders and stores, the 48-byte compressed G1 decoding, the
// EIP-2537 64-byte field element, Fp2 = Fp[u]/(u^2 + 1) over Fp381 with Fq2's interface, so curve.cuh's XYZZ formulas (and
// xyzz_scalar_mul) instantiate over the twist unchanged, the r P = O subgroup checks, and the workspace carver of the
// pairing-family calls.  The build has no -rdc: each translation unit keeps its own device copy of the __noinline__
// functions, and `inline` lets the host linker merge their host-side stubs.
#pragma once
#include "common.cuh"

namespace b200zk {

B2_D Fp381 load_be48(const uint8_t* in, uint32_t clear_top_mask) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(in);
  Fp381 v;
#pragma unroll
  for (int k = 0; k < 12; ++k) v.v[k] = __byte_perm(__ldg(w + 11 - k), 0, 0x0123);
  v.v[11] &= clear_top_mask;
  return v;
}

B2_D Fr381 load_be32(const uint8_t* in) {  // 32-byte big-endian integer -> canonical limbs
  const uint32_t* w = reinterpret_cast<const uint32_t*>(in);
  Fr381 v;
#pragma unroll
  for (int k = 0; k < 8; ++k) v.v[k] = __byte_perm(__ldg(w + 7 - k), 0, 0x0123);
  return v;
}

B2_D void store_be32(uint8_t* out, const Fr381& canonical) {  // load_be32's inverse (out 4-byte aligned)
  uint32_t* o = reinterpret_cast<uint32_t*>(out);
#pragma unroll
  for (int k = 0; k < 8; ++k) o[k] = __byte_perm(canonical.v[7 - k], 0, 0x0123);
}

B2_D Fp381 fp381_half() {
  Fp381 h;
#pragma unroll
  for (int k = 0; k < 12; ++k) h.v[k] = Fp381Cfg::half(k);
  return h;
}

// 48-byte compressed G1 point (ZCash form) -> native affine (identity = (0, 0)).  0 ok, B200ZK_ERR_NOT_IN_FIELD when
// x >= p, B200ZK_ERR_NOT_ON_CURVE when the flag bits are inconsistent or x^3 + 4 is not a square.  No subgroup check.
B2_D uint32_t bls_g1_decompress(const uint8_t* src, Affine<Fp381>* pt) {
  const uint8_t flags = src[0];
  const bool c_flag = flags & 0x80, inf_flag = flags & 0x40, sign_flag = flags & 0x20;
  *pt = {Fp381::zero(), Fp381::zero()};
  const Fp381 x = load_be48(src, 0x1fffffffu);
  if (!c_flag) return B200ZK_ERR_NOT_ON_CURVE;
  if (inf_flag) return (sign_flag || !x.is_zero()) ? (uint32_t)B200ZK_ERR_NOT_ON_CURVE : 0u;
  if (!Fp381::less(x, Fp381::modulus())) return B200ZK_ERR_NOT_IN_FIELD;
  const Fp381 xm = Fp381::to_mont(x);
  const Fp381 rhs = Fp381::add(Fp381::mul(Fp381::sqr(xm), xm), CurveB<Fp381>::b());
  Fp381 y = Fp381::sqrt_candidate(rhs);
  if (Fp381::sqr(y) != rhs) return B200ZK_ERR_NOT_ON_CURVE;  // x^3 + 4 is not a square: no such point
  const bool largest = Fp381::less(fp381_half(), Fp381::from_mont(y));
  if (largest != sign_flag) y = Fp381::neg(y);
  *pt = {xm, y};
  return 0;
}

// Fp2 = Fp[u]/(u^2 + 1) over the BLS12-381 base field; c0 = real, c1 = imaginary (Montgomery components)
struct Fp2_381 {
  Fp381 c0, c1;
  static B2_D Fp2_381 zero() { return {Fp381::zero(), Fp381::zero()}; }
  static B2_D Fp2_381 one() { return {Fp381::one(), Fp381::zero()}; }
  B2_D bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
  B2_D bool operator==(const Fp2_381& b) const { return c0 == b.c0 && c1 == b.c1; }
  B2_D bool operator!=(const Fp2_381& b) const { return !(*this == b); }
  static B2_D Fp2_381 add(const Fp2_381& a, const Fp2_381& b) { return {Fp381::add(a.c0, b.c0), Fp381::add(a.c1, b.c1)}; }
  static B2_D Fp2_381 sub(const Fp2_381& a, const Fp2_381& b) { return {Fp381::sub(a.c0, b.c0), Fp381::sub(a.c1, b.c1)}; }
  static B2_D Fp2_381 dbl(const Fp2_381& a) { return {Fp381::dbl(a.c0), Fp381::dbl(a.c1)}; }
  static B2_D Fp2_381 neg(const Fp2_381& a) { return {Fp381::neg(a.c0), Fp381::neg(a.c1)}; }
  static B2_D Fp2_381 conj(const Fp2_381& a) { return {a.c0, Fp381::neg(a.c1)}; }
  // Karatsuba: three base-field products (each a call to the one non-inlined Fp381::mul)
  static __device__ __noinline__ Fp2_381 mul(const Fp2_381& a, const Fp2_381& b) {
    const Fp381 t0 = Fp381::mul(a.c0, b.c0), t1 = Fp381::mul(a.c1, b.c1);
    const Fp381 s = Fp381::mul(Fp381::add(a.c0, a.c1), Fp381::add(b.c0, b.c1));
    return {Fp381::sub(t0, t1), Fp381::sub(Fp381::sub(s, t0), t1)};
  }
  static B2_D Fp2_381 sqr(const Fp2_381& a) {  // (c0 + c1)(c0 - c1), 2 c0 c1
    const Fp381 m = Fp381::mul(a.c0, a.c1);
    return {Fp381::mul(Fp381::add(a.c0, a.c1), Fp381::sub(a.c0, a.c1)), Fp381::dbl(m)};
  }
  static B2_D Fp2_381 mul2_sub(const Fp2_381& a, const Fp2_381& b, const Fp2_381& c, const Fp2_381& d) { return sub(mul(a, b), mul(c, d)); }
  static B2_D Fp2_381 scale(const Fp2_381& a, const Fp381& k) { return {Fp381::mul(a.c0, k), Fp381::mul(a.c1, k)}; }
  static B2_D Fp2_381 mul_xi(const Fp2_381& a) { return {Fp381::sub(a.c0, a.c1), Fp381::add(a.c0, a.c1)}; }  // * (1 + u)
  static __device__ __noinline__ Fp2_381 inv(const Fp2_381& a) {  // inv(0) = 0
    const Fp381 d = Fp381::inv(Fp381::add(Fp381::sqr(a.c0), Fp381::sqr(a.c1)));
    return {Fp381::mul(a.c0, d), Fp381::neg(Fp381::mul(a.c1, d))};
  }
  static B2_D Fp2_381 pow(const Fp2_381& a, const uint32_t* e) {  // e = 12 little-endian limbs
    Fp2_381 acc = one();
#pragma unroll 1
    for (int i = 32 * 12 - 1; i >= 0; --i) {
      acc = sqr(acc);
      if ((e[i >> 5] >> (i & 31)) & 1) acc = mul(acc, a);
    }
    return acc;
  }
  // a square root when a is a square (p = 3 mod 4; Adj and Rodriguez-Henriquez, "Square root computation over even
  // extension fields", Algorithm 9): a1 = a^((p-3)/4), alpha = a1^2 a = a^((p-1)/2), x0 = a1 a; x = u x0 when alpha = -1,
  // else (1 + alpha)^((p-1)/2) x0.  The caller checks x^2 == a.
  static __device__ __noinline__ Fp2_381 sqrt_candidate(const Fp2_381& a) {
    uint32_t e[12];
#pragma unroll
    for (int k = 0; k < 12; ++k) e[k] = Fp381Cfg::sqrt_exp(k);
    e[0] -= 1;  // (p+1)/4 - 1 = (p-3)/4; limb 0 of (p+1)/4 is 0xffffeaab: no borrow
    const Fp2_381 a1 = pow(a, e);
    const Fp2_381 x0 = mul(a1, a), alpha = mul(a1, x0);
#pragma unroll
    for (int k = 0; k < 12; ++k) e[k] = Fp381Cfg::half(k);
    if (alpha == neg(one())) return {Fp381::neg(x0.c1), x0.c0};  // u x0
    return mul(pow(add(one(), alpha), e), x0);
  }
};

template <> struct CurveB<Fp2_381> {
  static B2_D Fp2_381 b() { Fp381 four = Fp381::zero(); four.v[0] = 4; four = Fp381::to_mont(four); return {four, four}; }  // 4 (1 + u)
};

// ---- subgroup checks: r P = O (no endomorphism shortcuts) -------------------------------------------------------------
__device__ __noinline__ inline bool g1_in_subgroup(const Affine<Fp381>& p) {
  uint32_t k[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) k[j] = bls_r_limb(j);
  return xyzz_scalar_mul<Fp381>(k, p).is_inf();
}
__device__ __noinline__ inline bool g2_in_subgroup(const Affine<Fp2_381>& q) {
  uint32_t k[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) k[j] = bls_r_limb(j);
  return xyzz_scalar_mul<Fp2_381>(k, q).is_inf();
}

// EIP-2537 field element: 16 zero bytes, then 48 bytes big-endian below p
B2_D bool load_fp64(const uint8_t* src, Fp381* out) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(src);
  const uint32_t pad = __ldg(w) | __ldg(w + 1) | __ldg(w + 2) | __ldg(w + 3);
  *out = load_be48(src + 16, 0xffffffffu);
  return pad == 0 && Fp381::less(*out, Fp381::modulus());
}

// canonical limbs -> 48 bytes big-endian (out 4-byte aligned); load_be48's inverse
B2_D void store_be48(uint8_t* out, const Fp381& canonical) {
  uint32_t* w = reinterpret_cast<uint32_t*>(out);
#pragma unroll
  for (int k = 0; k < 12; ++k) w[11 - k] = __byte_perm(canonical.v[k], 0, 0x0123);
}

// native affine -> the 48-byte compressed form, bls_g1_decompress's inverse; the identity is 0xc0 | 0..0 (out 4-byte aligned)
B2_D void bls_g1_compress(uint8_t* out, const Affine<Fp381>& p) {
  if (p.is_inf()) {
    uint32_t* w = reinterpret_cast<uint32_t*>(out);
#pragma unroll
    for (int k = 0; k < 12; ++k) w[k] = 0;
    out[0] = 0xc0;
    return;
  }
  store_be48(out, Fp381::from_mont(p.x));
  out[0] |= 0x80 | (Fp381::less(fp381_half(), Fp381::from_mont(p.y)) ? 0x20 : 0x00);
}

}  // namespace b200zk
