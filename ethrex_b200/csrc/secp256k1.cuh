// secp256k1.cuh -- secp256k1 public-key recovery (ECDSA ECRECOVER) for one item per thread: the base field p =
// 2^256 - 2^32 - 977, the scalar field n, the curve y^2 = x^3 + 7 through curve.cuh's templates, and keccak256 of the
// recovered key.  Every function is __host__ __device__ and portable C++ (no inline PTX), so the tests compile this
// header for the host with nvcc and compare it with a Python oracle without a device; the kernel runs the same code.
//
// Semantics are libsecp256k1's (secp256k1_ecdsa_recover after RecoverableSignature::from_compact), the default path of
// the reference's Crypto::secp256k1_ecrecover; see secp_recover below for the order of the checks.
#pragma once
#include "curve.cuh"
#include "keccak.cuh"

namespace b200zk {

namespace secp {
// little-endian 32-bit limbs
B2_HD constexpr uint32_t P(int i) {  // p = 2^256 - 2^32 - 977
  constexpr uint32_t m[8] = {0xfffffc2fu, 0xfffffffeu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
  return m[i];
}
B2_HD constexpr uint32_t N(int i) {  // the group order n
  constexpr uint32_t m[8] = {0xd0364141u, 0xbfd25e8cu, 0xaf48a03bu, 0xbaaedce6u, 0xfffffffeu, 0xffffffffu, 0xffffffffu, 0xffffffffu};
  return m[i];
}
B2_HD constexpr uint32_t N_HALF(int i) {  // floor(n / 2): EIP-2's bound on s
  constexpr uint32_t m[8] = {0x681b20a0u, 0xdfe92f46u, 0x57a4501du, 0x5d576e73u, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x7fffffffu};
  return m[i];
}
B2_HD constexpr uint32_t P_MINUS_N(int i) {  // p - n: recids 2 and 3 need r < p - n, so that x = r + n < p
  constexpr uint32_t m[8] = {0x2fc9baeeu, 0x402da172u, 0x50b75fc4u, 0x45512319u, 0x00000001u, 0u, 0u, 0u};
  return m[i];
}
B2_HD constexpr uint32_t N_R1(int i) {  // 2^256 mod n
  constexpr uint32_t m[8] = {0x2fc9bebfu, 0x402da173u, 0x50b75fc4u, 0x45512319u, 0x00000001u, 0u, 0u, 0u};
  return m[i];
}
B2_HD constexpr uint32_t N_R2(int i) {  // 2^512 mod n
  constexpr uint32_t m[8] = {0x67d7d140u, 0x896cf214u, 0x0e7cf878u, 0x741496c2u, 0x5bcd07c6u, 0xe697f5e4u, 0x81c69bc5u, 0x9d671cd5u};
  return m[i];
}
constexpr uint32_t N_INV = 0x5588b13fu;  // -n^-1 mod 2^32
B2_HD constexpr uint32_t GX(int i) {
  constexpr uint32_t m[8] = {0x16f81798u, 0x59f2815bu, 0x2dce28d9u, 0x029bfcdbu, 0xce870b07u, 0x55a06295u, 0xf9dcbbacu, 0x79be667eu};
  return m[i];
}
B2_HD constexpr uint32_t GY(int i) {
  constexpr uint32_t m[8] = {0xfb10d4b8u, 0x9c47d08fu, 0xa6855419u, 0xfd17b448u, 0x0e1108a8u, 0x5da4fbfcu, 0x26a3c465u, 0x483ada77u};
  return m[i];
}

// r = a + b mod 2^256, returns the carry
B2_HD uint32_t add256(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) { c += (uint64_t)a[i] + b[i]; r[i] = (uint32_t)c; c >>= 32; }
  return (uint32_t)c;
}
// r = a - b mod 2^256, returns the borrow
B2_HD uint32_t sub256(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) { c = (uint64_t)a[i] - b[i] - c; r[i] = (uint32_t)c; c = (c >> 32) & 1; }
  return (uint32_t)c;
}
B2_HD bool less256(const uint32_t* a, const uint32_t* b) { uint32_t t[8]; return sub256(t, a, b) != 0; }
template <class K> B2_HD void load_const(uint32_t* r, K k) {
#pragma unroll
  for (int i = 0; i < 8; ++i) r[i] = k(i);
}
// 32 big-endian bytes -> little-endian limbs
B2_HD void load_be256(uint32_t* r, const uint8_t* b) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint8_t* w = b + 28 - 4 * i;
    r[i] = (uint32_t)w[0] << 24 | (uint32_t)w[1] << 16 | (uint32_t)w[2] << 8 | w[3];
  }
}
B2_HD void store_be256(uint8_t* b, const uint32_t* a) {
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    uint8_t* w = b + 28 - 4 * i;
    w[0] = (uint8_t)(a[i] >> 24); w[1] = (uint8_t)(a[i] >> 16); w[2] = (uint8_t)(a[i] >> 8); w[3] = (uint8_t)a[i];
  }
}

// t[0..15] = a * b (schoolbook).  Each step adds a 32x32 product, a limb and a carry: at most 2^64 - 1, so one 64-bit
// accumulator holds it.
B2_HD void mul512(uint32_t* t, const uint32_t* a, const uint32_t* b) {
#pragma unroll
  for (int i = 0; i < 16; ++i) t[i] = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    uint64_t c = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { c += (uint64_t)t[i + j] + (uint64_t)a[i] * b[j]; t[i + j] = (uint32_t)c; c >>= 32; }
    t[i + 8] = (uint32_t)c;
  }
}
// t[0..15] = a^2: the 28 cross products once, doubled, plus the 8 squares on the diagonal
B2_HD void sqr512(uint32_t* t, const uint32_t* a) {
#pragma unroll
  for (int i = 0; i < 16; ++i) t[i] = 0;
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    uint64_t c = 0;
#pragma unroll
    for (int j = i + 1; j < 8; ++j) { c += (uint64_t)t[i + j] + (uint64_t)a[i] * a[j]; t[i + j] = (uint32_t)c; c >>= 32; }
    t[i + 8] = (uint32_t)c;
  }
  // the cross sum is < 2^511, so doubling it loses nothing
#pragma unroll
  for (int i = 15; i > 0; --i) t[i] = t[i] << 1 | t[i - 1] >> 31;
  t[0] <<= 1;
  uint64_t c = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint64_t sq = (uint64_t)a[i] * a[i];
    c += (uint64_t)t[2 * i] + (uint32_t)sq; t[2 * i] = (uint32_t)c; c >>= 32;
    c += (uint64_t)t[2 * i + 1] + (sq >> 32); t[2 * i + 1] = (uint32_t)c; c >>= 32;
  }
}
}  // namespace secp

// ---- base field: canonical values 0 <= v < p, no Montgomery form --------------------------------------------------------
// p fills all 256 bits, so there is no headroom: add keeps the carry out of limb 7, and mul reduces a full 512-bit
// product through 2^256 = 2^32 + 977 (mod p).  to_mont / from_mont are the identity; they exist for curve.cuh.
struct SecpFp {
  uint32_t v[8];

  static B2_HD SecpFp zero() { SecpFp r; for (int i = 0; i < 8; ++i) r.v[i] = 0; return r; }
  static B2_HD SecpFp one() { SecpFp r = zero(); r.v[0] = 1; return r; }
  static B2_HD SecpFp modulus() { SecpFp r; secp::load_const(r.v, secp::P); return r; }
  B2_HD bool is_zero() const {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) o |= v[i];
    return o == 0;
  }
  B2_HD bool operator==(const SecpFp& b) const {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) o |= v[i] ^ b.v[i];
    return o == 0;
  }
  B2_HD bool operator!=(const SecpFp& b) const { return !(*this == b); }

  // a, b < p: the sum is < 2p < 2^257.  With the carry c, s + c 2^256 >= p exactly when c is set or s - p does not borrow.
  static B2_HD SecpFp add(const SecpFp& a, const SecpFp& b) {
    SecpFp s, t, m = modulus();
    const uint32_t c = secp::add256(s.v, a.v, b.v);
    const uint32_t bo = secp::sub256(t.v, s.v, m.v);
    return (c | !bo) ? t : s;
  }
  // a, b < p: on a borrow a - b + 2^256 + p wraps to a - b + p < p
  static B2_HD SecpFp sub(const SecpFp& a, const SecpFp& b) {
    SecpFp d, m = modulus();
    if (secp::sub256(d.v, a.v, b.v)) secp::add256(d.v, d.v, m.v);
    return d;
  }
  static B2_HD SecpFp dbl(const SecpFp& a) { return add(a, a); }
  static B2_HD SecpFp neg(const SecpFp& a) { return a.is_zero() ? a : sub(zero(), a); }

  // t < 2^512 (any product of 256-bit values) -> t mod p.  t = lo + 2^256 hi = lo + (2^32 + 977) hi (mod p):
  //   fold 1: lo + 977 hi + (hi << 32) < 2^256 + 2^32 (978 (2^256 - 1)) < 2^256 (1 + 2^42): nine limbs, the ninth c1 < 2^43;
  //   fold 2: r + c1 (2^32 + 977) < 2^256 + 2^76: at most one carry d out of limb 7; when d = 1, r < 2^76;
  //   fold 3: r + d (2^32 + 977) with r < 2^76 cannot carry again.  Then r < 2^256 < 2p: one conditional subtraction.
  static B2_HD SecpFp reduce512(const uint32_t* t) {
    uint32_t r[8];
    uint64_t c = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      c += (uint64_t)t[i] + (uint64_t)t[8 + i] * 977u + (i ? t[7 + i] : 0u);
      r[i] = (uint32_t)c;
      c >>= 32;
    }
    c += t[15];  // hi << 32 pushes hi's top limb to column 8
    uint64_t d = (uint64_t)r[0] + c * 977u;
    r[0] = (uint32_t)d; d >>= 32;
    d += (uint64_t)r[1] + c;
    r[1] = (uint32_t)d; d >>= 32;
#pragma unroll
    for (int i = 2; i < 8; ++i) { d += r[i]; r[i] = (uint32_t)d; d >>= 32; }
    uint64_t e = (uint64_t)r[0] + d * 977u;
    r[0] = (uint32_t)e; e >>= 32;
    e += (uint64_t)r[1] + d;
    r[1] = (uint32_t)e; e >>= 32;
#pragma unroll
    for (int i = 2; i < 8; ++i) { e += r[i]; r[i] = (uint32_t)e; e >>= 32; }
    SecpFp s, u, m = modulus();
#pragma unroll
    for (int i = 0; i < 8; ++i) s.v[i] = r[i];
    return secp::sub256(u.v, s.v, m.v) ? s : u;
  }
  // any 256-bit inputs (reduce512 needs none of the bounds Fe relies on); the result is < p
  static B2_HD SecpFp mul(const SecpFp& a, const SecpFp& b) { uint32_t t[16]; secp::mul512(t, a.v, b.v); return reduce512(t); }
  static B2_HD SecpFp sqr(const SecpFp& a) { uint32_t t[16]; secp::sqr512(t, a.v); return reduce512(t); }
  static B2_HD SecpFp mul2_sub(const SecpFp& a, const SecpFp& b, const SecpFp& c, const SecpFp& d) { return sub(mul(a, b), mul(c, d)); }
  static B2_HD SecpFp to_mont(const SecpFp& a) { return a; }
  static B2_HD SecpFp from_mont(const SecpFp& a) { return a; }
  // a^e, e = 256-bit little-endian limbs (square-and-multiply, MSB first)
  static B2_HD SecpFp pow(const SecpFp& a, const uint32_t* e) {
    SecpFp acc = one();
    for (int i = 255; i >= 0; --i) {
      acc = sqr(acc);
      if ((e[i >> 5] >> (i & 31)) & 1) acc = mul(acc, a);
    }
    return acc;
  }
  static B2_HD SecpFp inv(const SecpFp& a) {  // Fermat: a^(p-2); inv(0) = 0
    uint32_t e[8];
    secp::load_const(e, secp::P);
    e[0] -= 2;  // p ends in ...fc2f: no borrow
    return pow(a, e);
  }
  // a square root of a when one exists: p = 3 (mod 4), so a^((p+1)/4) squares back to a exactly when a is a residue
  static B2_HD bool sqrt(const SecpFp& a, SecpFp* r) {
    const uint32_t e[8] = {0xbfffff0cu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0xffffffffu, 0x3fffffffu};
    *r = pow(a, e);
    return sqr(*r) == a;
  }
};

template <> struct CurveB<SecpFp> {
  static B2_HD SecpFp b() { SecpFp s = SecpFp::zero(); s.v[0] = 7; return s; }  // y^2 = x^3 + 7
};

// ---- scalar field mod n: Montgomery (R = 2^256), a few operations per signature, so plain CIOS ---------------------------
struct SecpFn {
  uint32_t v[8];
  // a, b < n -> a b / 2^256 mod n.  CIOS: the running total stays < 2n < 2^257, held in t[0..8] plus the carry t[9],
  // so one conditional subtraction (taken also when t[8] is set) canonicalises it.
  static B2_HD SecpFn mul(const SecpFn& a, const SecpFn& b) {
    uint32_t t[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int i = 0; i < 8; ++i) {
      uint64_t c = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { c += (uint64_t)t[j] + (uint64_t)a.v[j] * b.v[i]; t[j] = (uint32_t)c; c >>= 32; }
      c += t[8]; t[8] = (uint32_t)c; t[9] = (uint32_t)(c >> 32);
      const uint32_t m = t[0] * secp::N_INV;
      c = ((uint64_t)t[0] + (uint64_t)m * secp::N(0)) >> 32;
#pragma unroll
      for (int j = 1; j < 8; ++j) { c += (uint64_t)t[j] + (uint64_t)m * secp::N(j); t[j - 1] = (uint32_t)c; c >>= 32; }
      c += t[8]; t[7] = (uint32_t)c; c >>= 32;
      t[8] = t[9] + (uint32_t)c;
    }
    SecpFn r, s, n;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.v[i] = t[i];
    secp::load_const(n.v, secp::N);
    const uint32_t bo = secp::sub256(s.v, r.v, n.v);
    return (t[8] | !bo) ? s : r;
  }
  static B2_HD SecpFn from_canonical(const uint32_t* a) {  // a < n
    SecpFn x, r2;
#pragma unroll
    for (int i = 0; i < 8; ++i) x.v[i] = a[i];
    secp::load_const(r2.v, secp::N_R2);
    return mul(x, r2);
  }
  B2_HD void to_canonical(uint32_t* out) const {
    SecpFn one = {{1, 0, 0, 0, 0, 0, 0, 0}};
    const SecpFn r = mul(*this, one);
#pragma unroll
    for (int i = 0; i < 8; ++i) out[i] = r.v[i];
  }
  static B2_HD SecpFn neg(const SecpFn& a) {
    SecpFn r, n;
    secp::load_const(n.v, secp::N);
    secp::sub256(r.v, n.v, a.v);
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) o |= a.v[i];
    return o ? r : a;
  }
  static B2_HD SecpFn inv(const SecpFn& a) {  // Fermat: a^(n-2), Montgomery in and out
    uint32_t e[8];
    secp::load_const(e, secp::N);
    e[0] -= 2;  // n ends in ...4141: no borrow
    SecpFn acc;
    secp::load_const(acc.v, secp::N_R1);
    for (int i = 255; i >= 0; --i) {
      acc = mul(acc, acc);
      if ((e[i >> 5] >> (i & 31)) & 1) acc = mul(acc, a);
    }
    return acc;
  }
};

// ---- keccak256: keccak.cuh (shared with the PLONK transcript) ----------------------------------------------------------

// ---- recovery; its G table, wNAF and ladder below are shared with P-256 (secp256r1.cuh) -----------------------------------
constexpr uint32_t kSecpLowS = 1;  // B200ZK_ECRECOVER_LOW_S
enum : uint32_t { kEcrecOk = 0, kEcrecInvalidSignature = 2, kEcrecRecoveryFailed = 3, kEcrecInvalidRecoveryId = 4 };
// fixed-base window of the G term: 12-bit digits of u1, 22 mixed additions.  Measured against 4 and 8 bits (DESIGN.md
// section 4.10): registers are the same, and 12 bits is the fastest at large batches
constexpr int kSecpGWindow = 12;
constexpr int kSecpGTable = (1 << kSecpGWindow) - 1;         // table[d - 1] = d G, d = 1 .. 4095 (affine, 256 KB)
constexpr int kSecpRWindow = 5;                              // wNAF width of the R term: digits odd, |d| < 16
constexpr int kSecpRTable = 1 << (kSecpRWindow - 2);         // R, 3R, .., 15R

// an entry of the affine table the G term reads: table[d - 1] = d G
template <class F> B2_HD Affine<F> ecdsa_g_multiple(const Affine<F>& g, uint32_t d) {
  const uint32_t k[8] = {d, 0, 0, 0, 0, 0, 0, 0};
  return xyzz_to_affine(xyzz_scalar_mul(k, g));
}
B2_HD Affine<SecpFp> secp_g_multiple(uint32_t d) {
  Affine<SecpFp> g;
  secp::load_const(g.x.v, secp::GX);
  secp::load_const(g.y.v, secp::GY);
  return ecdsa_g_multiple(g, d);
}

// width-5 NAF of k < 2^256: k = sum naf[i] 2^i, every nonzero digit odd with |digit| < 16; 257 digits
B2_HD void secp_wnaf(const uint32_t* k, int8_t* naf) {
  uint32_t w[9];
#pragma unroll
  for (int i = 0; i < 8; ++i) w[i] = k[i];
  w[8] = 0;
  for (int i = 0; i <= 256; ++i) {
    int d = 0;
    if (w[0] & 1) {
      d = (int)(w[0] & 31);
      if (d >= 16) d -= 32;
      // w -= d: the low five bits of w are d's, so a positive d clears them without a borrow, a negative one carries
      uint64_t c = (uint64_t)w[0] - (int64_t)d;
      w[0] = (uint32_t)c;
      c >>= 32;
      for (int j = 1; j < 9 && c; ++j) { c += w[j]; w[j] = (uint32_t)c; c >>= 32; }
    }
    naf[i] = (int8_t)d;
#pragma unroll
    for (int j = 0; j < 8; ++j) w[j] = w[j] >> 1 | w[j + 1] << 31;
    w[8] >>= 1;
  }
}

// u1 G + u2 R in one MSB-first loop: one shared doubling per bit (257 steps, the first on the identity, so at most 256
// doublings), an XYZZ addition of +-(odd multiple of R) per nonzero wNAF digit of u2, and a mixed addition of
// gtab[w - 1] per nonzero window w of u1 at the window's lowest bit.  r is a curve point other than the identity; the
// curve enters only through the field F (and its CurveA / CurveB).
template <class F> B2_HD XYZZ<F> secp_lincomb(const uint32_t* u1, const uint32_t* u2, const Affine<F>& r, const Affine<F>* gtab) {
  XYZZ<F> rt[kSecpRTable];
  rt[0] = xyzz_from_affine(r);
  const XYZZ<F> r2 = xyzz_mdbl(r.x, r.y);
  for (int i = 1; i < kSecpRTable; ++i) { rt[i] = rt[i - 1]; xyzz_add(rt[i], r2); }
  int8_t naf[257];
  secp_wnaf(u2, naf);
  XYZZ<F> acc = XYZZ<F>::identity();
#pragma unroll 1
  for (int i = 256; i >= 0; --i) {
    acc = xyzz_dbl(acc);
    const int d = naf[i];
    if (d) {
      XYZZ<F> q = rt[(d < 0 ? -d : d) >> 1];
      if (d < 0) q.y = F::neg(q.y);
      xyzz_add(acc, q);
    }
    if (i % kSecpGWindow == 0 && i < 256) {
      const uint64_t two = u1[i >> 5] | (i < 224 ? (uint64_t)u1[(i >> 5) + 1] << 32 : 0);  // a window may cross a limb
      const uint32_t w = (uint32_t)(two >> (i & 31)) & ((1u << kSecpGWindow) - 1);
      if (w) {
        const Affine<F> g = gtab[w - 1];
        xyzz_add_mixed(acc, g.x, g.y);
      }
    }
  }
  return acc;
}

// One ECRECOVER item: sig = r (32 B BE) | s (32 B BE) | recid, msg = 32-byte hash.  out = keccak256(X | Y) of the
// recovered key, or zero bytes when the status is not 0.  Checks in order, the first failure decides:
//   1. flags & kSecpLowS and s > n/2              -> 2 (EIP-2, Crypto::recover_signer)
//   2. recid > 3                                   -> 4
//   3. r >= n or s >= n                            -> 2 (from_compact's overflow check)
//   4. r = 0 or s = 0; recid 2/3 with r >= p - n;
//      x (r, or r + n for recids 2/3) with no curve point; Q = O    -> 3
// Q = r^-1 (s R - z G), R = (x, y) with y's parity recid & 1, z = msg mod n.
B2_HD uint32_t secp_recover(const uint8_t* sig, const uint8_t* msg, uint32_t flags, const Affine<SecpFp>* gtab, uint8_t* out) {
#pragma unroll
  for (int i = 0; i < 32; ++i) out[i] = 0;
  uint32_t r[8], s[8], z[8], k[8];
  secp::load_be256(r, sig);
  secp::load_be256(s, sig + 32);
  const uint32_t recid = sig[64];
  secp::load_const(k, secp::N_HALF);
  if ((flags & kSecpLowS) && secp::less256(k, s)) return kEcrecInvalidSignature;
  if (recid > 3) return kEcrecInvalidRecoveryId;
  secp::load_const(k, secp::N);
  if (!secp::less256(r, k) || !secp::less256(s, k)) return kEcrecInvalidSignature;
  uint32_t rz = 0, sz = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) { rz |= r[i]; sz |= s[i]; }
  if (!rz || !sz) return kEcrecRecoveryFailed;
  SecpFp x;
#pragma unroll
  for (int i = 0; i < 8; ++i) x.v[i] = r[i];
  if (recid & 2) {
    uint32_t pn[8];
    secp::load_const(pn, secp::P_MINUS_N);
    if (!secp::less256(r, pn)) return kEcrecRecoveryFailed;
    secp::add256(x.v, r, k);  // r + n < p
  }
  Affine<SecpFp> R;
  R.x = x;
  if (!SecpFp::sqrt(SecpFp::add(SecpFp::mul(SecpFp::sqr(x), x), CurveB<SecpFp>::b()), &R.y)) return kEcrecRecoveryFailed;
  if ((R.y.v[0] & 1) != (recid & 1)) R.y = SecpFp::neg(R.y);  // y != 0: n is odd, so there is no point of order 2
  // u1 = -z / r, u2 = s / r (mod n)
  secp::load_be256(z, msg);
  uint32_t zr[8];
  if (!secp::sub256(zr, z, k)) {  // z < 2^256 < 2n: one subtraction reduces it
#pragma unroll
    for (int i = 0; i < 8; ++i) z[i] = zr[i];
  }
  const SecpFn ri = SecpFn::inv(SecpFn::from_canonical(r));
  uint32_t u1[8], u2[8];
  SecpFn::neg(SecpFn::mul(SecpFn::from_canonical(z), ri)).to_canonical(u1);
  SecpFn::mul(SecpFn::from_canonical(s), ri).to_canonical(u2);
  const XYZZ<SecpFp> q = secp_lincomb(u1, u2, R, gtab);
  if (q.is_inf()) return kEcrecRecoveryFailed;
  const Affine<SecpFp> a = xyzz_to_affine(q);
  uint8_t key[64];
  secp::store_be256(key, a.x.v);
  secp::store_be256(key + 32, a.y.v);
  keccak256_64(key, out);
  return kEcrecOk;
}

}  // namespace b200zk
