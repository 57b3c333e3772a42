// bls381.cuh -- BLS12-381 base field Fp (381 bits, 12 x 32-bit limbs, Montgomery R = 2^384) and the G1 byte formats, for
// the one place the L2 pipeline commits over this curve: EIP-4844 blob commitments,
//   /root/reference/crates/common/crypto/kzg.rs:259-272   blob_to_kzg_commitment_and_proof (c_kzg blob_to_kzg_commitment)
//   /root/reference/crates/common/types/blobs_bundle.rs:90-118   BlobsBundle::create_from_blobs
//   /root/reference/crates/l2/sequencer/l1_committer.rs:1488-1521   the committer's "commit" step
// (SURVEY.md section 8f row 3).  The commitment is a 4096-point G1 MSM over the trusted setup in Lagrange form.
//
// The field is the generic-width sibling of field.cuh's Fe: the same interface (zero / one / add / sub / dbl / neg / mul /
// sqr / mul2_sub / inv / is_zero / ==), so curve.cuh's XYZZ formulas and every MSM kernel of msm.cu instantiate over it
// unchanged.  A 4096-point MSM is latency bound (SURVEY.md 8f: "small n, modest win"), so the product is a plain
// operand-scanning CIOS on 64-bit accumulators (IMAD.WIDE after ptxas), not the hand-scheduled carry chains of Fe.
#pragma once
#include "field.cuh"

namespace b200zk {

struct Fp381Cfg {
  static constexpr int N = 12;
  // p = 0x1a0111ea397fe69a4b1ba7b6434bacd764774b84f38512bf6730d2a0f6b0f6241eabfffeb153ffffb9feffffffffaaab
  static B2_HD constexpr uint32_t mod(int i) {
    constexpr uint32_t m[12] = {0xffffaaabu, 0xb9feffffu, 0xb153ffffu, 0x1eabfffeu, 0xf6b0f624u, 0x6730d2a0u, 0xf38512bfu, 0x64774b84u, 0x434bacd7u, 0x4b1ba7b6u, 0x397fe69au, 0x1a0111eau};
    return m[i];
  }
  static B2_HD constexpr uint32_t r1(int i) {  // 2^384 mod p
    constexpr uint32_t m[12] = {0x0002fffdu, 0x76090000u, 0xc40c0002u, 0xebf4000bu, 0x53c758bau, 0x5f489857u, 0x70525745u, 0x77ce5853u, 0xa256ec6du, 0x5c071a97u, 0xfa80e493u, 0x15f65ec3u};
    return m[i];
  }
  static B2_HD constexpr uint32_t r2(int i) {  // 2^768 mod p
    constexpr uint32_t m[12] = {0x1c341746u, 0xf4df1f34u, 0x09d104f1u, 0x0a76e6a6u, 0x4c95b6d5u, 0x8de5476cu, 0x939d83c0u, 0x67eb88a9u, 0xb519952du, 0x9a793e85u, 0x92cae3aau, 0x11988fe5u};
    return m[i];
  }
  static B2_HD constexpr uint32_t sqrt_exp(int i) {  // (p + 1) / 4: p = 3 mod 4, so sqrt(a) = a^((p+1)/4) when a is a square
    constexpr uint32_t m[12] = {0xffffeaabu, 0xee7fbfffu, 0xac54ffffu, 0x07aaffffu, 0x3dac3d89u, 0xd9cc34a8u, 0x3ce144afu, 0xd91dd2e1u, 0x90d2eb35u, 0x92c6e9edu, 0x8e5ff9a6u, 0x0680447au};
    return m[i];
  }
  static B2_HD constexpr uint32_t half(int i) {  // (p - 1) / 2: y is "lexicographically largest" when y > (p-1)/2
    constexpr uint32_t m[12] = {0xffffd555u, 0xdcff7fffu, 0x58a9ffffu, 0x0f55ffffu, 0x7b587b12u, 0xb3986950u, 0x79c2895fu, 0xb23ba5c2u, 0x21a5d66bu, 0x258dd3dbu, 0x1cbff34du, 0x0d0088f5u};
    return m[i];
  }
  static constexpr uint32_t INV = 0xfffcfffdu;  // -p^-1 mod 2^32
};

// BLS12-381 scalar field modulus (255 bits): blob field elements must be below it (c-kzg: bytes_to_bls_field)
B2_HD constexpr uint32_t bls_r_limb(int i) {
  constexpr uint32_t m[8] = {0x00000001u, 0xffffffffu, 0xfffe5bfeu, 0x53bda402u, 0x09a1d805u, 0x3339d808u, 0x299d7d48u, 0x73eda753u};
  return m[i];
}

template <class Cfg>
struct FeBig {
  static constexpr int N = Cfg::N;
  uint32_t v[N];

  static B2_HD FeBig zero() { FeBig r; for (int i = 0; i < N; ++i) r.v[i] = 0; return r; }
  static B2_HD FeBig one() { FeBig r; for (int i = 0; i < N; ++i) r.v[i] = Cfg::r1(i); return r; }
  static B2_HD FeBig rsquared() { FeBig r; for (int i = 0; i < N; ++i) r.v[i] = Cfg::r2(i); return r; }
  static B2_HD FeBig modulus() { FeBig r; for (int i = 0; i < N; ++i) r.v[i] = Cfg::mod(i); return r; }
  B2_HD bool is_zero() const {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) o |= v[i];
    return o == 0;
  }
  B2_HD bool operator==(const FeBig& b) const {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) o |= v[i] ^ b.v[i];
    return o == 0;
  }
  B2_HD bool operator!=(const FeBig& b) const { return !(*this == b); }

  // r = a - b, returns the borrow (0 / 1)
  static B2_D uint32_t sub_limbs(uint32_t* r, const uint32_t* a, const uint32_t* b) {
    uint64_t br = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      uint64_t d = (uint64_t)a[i] - b[i] - br;
      r[i] = (uint32_t)d;
      br = (d >> 32) & 1u;
    }
    return (uint32_t)br;
  }
  static B2_D bool less(const FeBig& a, const FeBig& b) { uint32_t t[N]; return sub_limbs(t, a.v, b.v) != 0; }
  static B2_D FeBig reduce_once(const FeBig& a) {  // a < 2p -> a mod p
    FeBig t;
    const uint32_t borrow = sub_limbs(t.v, a.v, modulus().v);
    FeBig r;
#pragma unroll
    for (int i = 0; i < N; ++i) r.v[i] = borrow ? a.v[i] : t.v[i];
    return r;
  }
  static B2_D FeBig add(const FeBig& a, const FeBig& b) {  // 2p < 2^384 and 2r < 2^256: no carry out
    FeBig s;
    uint64_t c = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) { uint64_t t = (uint64_t)a.v[i] + b.v[i] + c; s.v[i] = (uint32_t)t; c = t >> 32; }
    return reduce_once(s);
  }
  static B2_D FeBig sub(const FeBig& a, const FeBig& b) {
    FeBig d;
    const uint32_t borrow = sub_limbs(d.v, a.v, b.v);
    uint64_t c = 0;
    FeBig r;
#pragma unroll
    for (int i = 0; i < N; ++i) { uint64_t t = (uint64_t)d.v[i] + (borrow ? Cfg::mod(i) : 0u) + c; r.v[i] = (uint32_t)t; c = t >> 32; }
    return r;
  }
  static B2_D FeBig dbl(const FeBig& a) { return add(a, a); }
  static B2_D FeBig neg(const FeBig& a) { return a.is_zero() ? a : sub(zero(), a); }

  // Montgomery product a * b / 2^(32 N) mod p: coarsely integrated operand scanning.  NOT inlined: one copy of the 2 x 144
  // multiply-adds per kernel instead of one per call site (the MSM kernels call it ~12 times per addition; inlining them
  // cost 10 minutes of compile time for nothing -- a 4096-point MSM is latency bound)
  static __device__ __noinline__ FeBig mul(const FeBig& a, const FeBig& b) {
    uint32_t t[N + 2];
#pragma unroll
    for (int i = 0; i < N + 2; ++i) t[i] = 0;
#pragma unroll
    for (int i = 0; i < N; ++i) {
      uint64_t c = 0;
#pragma unroll
      for (int j = 0; j < N; ++j) { uint64_t s = (uint64_t)a.v[j] * b.v[i] + t[j] + c; t[j] = (uint32_t)s; c = s >> 32; }
      uint64_t s = (uint64_t)t[N] + c;
      t[N] = (uint32_t)s; t[N + 1] = (uint32_t)(s >> 32);
      const uint32_t m = t[0] * Cfg::INV;
      c = ((uint64_t)m * Cfg::mod(0) + t[0]) >> 32;
#pragma unroll
      for (int j = 1; j < N; ++j) { uint64_t u = (uint64_t)m * Cfg::mod(j) + t[j] + c; t[j - 1] = (uint32_t)u; c = u >> 32; }
      s = (uint64_t)t[N] + c;
      t[N - 1] = (uint32_t)s;
      t[N] = t[N + 1] + (uint32_t)(s >> 32);
    }
    FeBig r;
#pragma unroll
    for (int i = 0; i < N; ++i) r.v[i] = t[i];
    return reduce_once(r);  // inputs < p => value < 2p, and t[N] == 0 (2p < 2^(32 N) for both moduli)
  }
  static B2_D FeBig sqr(const FeBig& a) { return mul(a, a); }
  static B2_D FeBig mul2_sub(const FeBig& a, const FeBig& b, const FeBig& c, const FeBig& d) { return sub(mul(a, b), mul(c, d)); }
  static B2_D FeBig to_mont(const FeBig& canonical) { return mul(canonical, rsquared()); }
  static B2_D FeBig from_mont(const FeBig& a) { FeBig o = zero(); o.v[0] = 1; return mul(a, o); }
  // a^e, e = N little-endian limbs
  static B2_D FeBig pow(const FeBig& a, const uint32_t* e) {
    FeBig acc = one();
#pragma unroll 1
    for (int i = 32 * N - 1; i >= 0; --i) {
      acc = sqr(acc);
      if ((e[i >> 5] >> (i & 31)) & 1) acc = mul(acc, a);
    }
    return acc;
  }
  static B2_D FeBig inv(const FeBig& a) {  // Fermat; inv(0) = 0
    uint32_t e[N];
    uint32_t br = 2;  // e = modulus - 2, borrow propagated: r ends in ...00000001
#pragma unroll
    for (int i = 0; i < N; ++i) { e[i] = Cfg::mod(i) - br; br = Cfg::mod(i) < br ? 1u : 0u; }
    return pow(a, e);
  }
  static B2_D FeBig sqrt_candidate(const FeBig& a) {  // a^((p+1)/4)
    uint32_t e[N];
#pragma unroll
    for (int i = 0; i < N; ++i) e[i] = Cfg::sqrt_exp(i);
    return pow(a, e);
  }
};

typedef FeBig<Fp381Cfg> Fp381;

// BLS12-381 scalar field Fr (255 bits, 8 x 32-bit limbs, Montgomery R = 2^256): the field blobs are polynomials over, for
// the EIP-4844 proof (evaluation at z and the quotient (p(X) - y) / (X - z)).  2r < 2^256, so FeBig's add and mul bounds hold.
struct Fr381Cfg {
  static constexpr int N = 8;
  static B2_HD constexpr uint32_t mod(int i) { return bls_r_limb(i); }
  static B2_HD constexpr uint32_t r1(int i) {  // 2^256 mod r
    constexpr uint32_t m[8] = {0xfffffffeu, 0x00000001u, 0x00034802u, 0x5884b7fau, 0xecbc4ff5u, 0x998c4fefu, 0xacc5056fu, 0x1824b159u};
    return m[i];
  }
  static B2_HD constexpr uint32_t r2(int i) {  // 2^512 mod r
    constexpr uint32_t m[8] = {0xf3f29c6du, 0xc999e990u, 0x87925c23u, 0x2b6cedcbu, 0x7254398fu, 0x05d31496u, 0x9f59ff11u, 0x0748d9d9u};
    return m[i];
  }
  static constexpr uint32_t INV = 0xffffffffu;  // -r^-1 mod 2^32 (r = 1 mod 2^32)
};

typedef FeBig<Fr381Cfg> Fr381;

}  // namespace b200zk
