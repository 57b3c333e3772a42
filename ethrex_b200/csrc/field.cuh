// field.cuh -- 254-bit prime-field arithmetic for sm_90a: BN254 base field Fq and scalar field Fr,
// Montgomery form with R = 2^256, eight 32-bit limbs per element (little-endian; the same bytes as
// ark-ff's Fp256<MontBackend> 4x64 in-memory form on a little-endian host).
//
// Replaces (for the hot path) the field arithmetic ethrex reaches through ark-ff 0.5.0 /
// ark-bn254 0.5.0 (/root/reference/Cargo.lock, call sites
// /root/reference/crates/common/crypto/provider.rs:201-330).
//
// The product is an operand-scanning Montgomery multiplication whose partial products are kept in
// two interleaved accumulators ("even" columns 0,2,4,6 and "odd" columns 1,3,5,7) so that every
// mad.lo.cc/madc.hi.cc pair lands on a 64-bit aligned column pair and each accumulator is ONE
// uninterrupted carry chain; ptxas turns each lo/hi pair into a single IMAD.WIDE.U32(.X).  Dividing
// by 2^32 after each round swaps the roles of the two accumulators.  Each carry chain is a single
// asm statement so the compiler can never separate a producer of CC from its consumer.
#pragma once
#include <cstdint>

#define B2_HD __host__ __device__ __forceinline__
#define B2_D __device__ __forceinline__

namespace b200zk {

struct FqCfg {
  // p = 0x30644e72e131a029b85045b68181585d97816a916871ca8d3c208c16d87cfd47
  // (ALT_BN128_PRIME, /root/reference/crates/vm/levm/src/precompiles.rs:746-751)
  static B2_HD constexpr uint32_t mod(int i) {
    constexpr uint32_t m[8] = {0xd87cfd47u, 0x3c208c16u, 0x6871ca8du, 0x97816a91u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
    return m[i];
  }
  static B2_HD constexpr uint32_t r1(int i) {  // R mod p
    constexpr uint32_t m[8] = {0xc58f0d9du, 0xd35d438du, 0xf5c70b3du, 0x0a78eb28u, 0x7879462cu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
    return m[i];
  }
  static B2_HD constexpr uint32_t r2(int i) {  // R^2 mod p
    constexpr uint32_t m[8] = {0x538afa89u, 0xf32cfc5bu, 0xd44501fbu, 0xb5e71911u, 0x0a417ff6u, 0x47ab1effu, 0xcab8351fu, 0x06d89f71u};
    return m[i];
  }
  static constexpr uint32_t INV = 0xe4866389u;  // -p^-1 mod 2^32
};

struct FrCfg {
  // r = 0x30644e72e131a029b85045b68181585d2833e84879b9709143e1f593f0000001
  static B2_HD constexpr uint32_t mod(int i) {
    constexpr uint32_t m[8] = {0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
    return m[i];
  }
  static B2_HD constexpr uint32_t r1(int i) {
    constexpr uint32_t m[8] = {0x4ffffffbu, 0xac96341cu, 0x9f60cd29u, 0x36fc7695u, 0x7879462eu, 0x666ea36fu, 0x9a07df2fu, 0x0e0a77c1u};
    return m[i];
  }
  static B2_HD constexpr uint32_t r2(int i) {
    constexpr uint32_t m[8] = {0xae216da7u, 0x1bb8e645u, 0xe35c59e3u, 0x53fe3ab1u, 0x53bb8085u, 0x8c49833du, 0x7f4e44a5u, 0x0216d0b1u};
    return m[i];
  }
  static constexpr uint32_t INV = 0xefffffffu;  // -r^-1 mod 2^32
};

// ------------------------------------------------------------------------------------------------
// carry-chain primitives (device only).  Every chain is one asm statement.
namespace detail {

// x[0..7] += a_even * b  (a0,a2,a4,a6 at columns 0,2,4,6);  carry out of column 7 is added to `top`.
B2_D void mad_even(uint32_t* x, uint32_t& top, uint32_t a0, uint32_t a2, uint32_t a4, uint32_t a6, uint32_t b) {
  asm("mad.lo.cc.u32  %0, %9,  %13, %0;\n\t"
      "madc.hi.cc.u32 %1, %9,  %13, %1;\n\t"
      "madc.lo.cc.u32 %2, %10, %13, %2;\n\t"
      "madc.hi.cc.u32 %3, %10, %13, %3;\n\t"
      "madc.lo.cc.u32 %4, %11, %13, %4;\n\t"
      "madc.hi.cc.u32 %5, %11, %13, %5;\n\t"
      "madc.lo.cc.u32 %6, %12, %13, %6;\n\t"
      "madc.hi.cc.u32 %7, %12, %13, %7;\n\t"
      "addc.u32       %8, %8, 0;"
      : "+r"(x[0]), "+r"(x[1]), "+r"(x[2]), "+r"(x[3]), "+r"(x[4]), "+r"(x[5]), "+r"(x[6]), "+r"(x[7]), "+r"(top)
      : "r"(a0), "r"(a2), "r"(a4), "r"(a6), "r"(b));
}

// y[0..7] += a_odd * b  (a1,a3,a5,a7; y[k] is column k+1).  No carry out (see bound in mont_mul).
B2_D void mad_odd(uint32_t* y, uint32_t a1, uint32_t a3, uint32_t a5, uint32_t a7, uint32_t b) {
  asm("mad.lo.cc.u32  %0, %8,  %12, %0;\n\t"
      "madc.hi.cc.u32 %1, %8,  %12, %1;\n\t"
      "madc.lo.cc.u32 %2, %9,  %12, %2;\n\t"
      "madc.hi.cc.u32 %3, %9,  %12, %3;\n\t"
      "madc.lo.cc.u32 %4, %10, %12, %4;\n\t"
      "madc.hi.cc.u32 %5, %10, %12, %5;\n\t"
      "madc.lo.cc.u32 %6, %11, %12, %6;\n\t"
      "madc.hi.u32    %7, %11, %12, %7;"
      : "+r"(y[0]), "+r"(y[1]), "+r"(y[2]), "+r"(y[3]), "+r"(y[4]), "+r"(y[5]), "+r"(y[6]), "+r"(y[7])
      : "r"(a1), "r"(a3), "r"(a5), "r"(a7), "r"(b));
}

// Role swap after the division by 2^32.  `x` was the odd accumulator (now column-0 aligned), `e` was
// the even accumulator whose column 0 is zero: its column 1 is folded into x[0] and the carry runs on
// into the new odd accumulator e'[k] = e[k+2] + (a_odd * b) (written in place over e).
B2_D void shift_mad_odd(uint32_t* e, uint32_t& x0, uint32_t a1, uint32_t a3, uint32_t a5, uint32_t a7, uint32_t b) {
  asm("add.cc.u32     %8, %8, %1;\n\t"
      "madc.lo.cc.u32 %0, %9,  %13, %2;\n\t"
      "madc.hi.cc.u32 %1, %9,  %13, %3;\n\t"
      "madc.lo.cc.u32 %2, %10, %13, %4;\n\t"
      "madc.hi.cc.u32 %3, %10, %13, %5;\n\t"
      "madc.lo.cc.u32 %4, %11, %13, %6;\n\t"
      "madc.hi.cc.u32 %5, %11, %13, %7;\n\t"
      "madc.lo.cc.u32 %6, %12, %13, 0;\n\t"
      "madc.hi.u32    %7, %12, %13, 0;"
      : "+r"(e[0]), "+r"(e[1]), "+r"(e[2]), "+r"(e[3]), "+r"(e[4]), "+r"(e[5]), "+r"(e[6]), "+r"(e[7]), "+r"(x0)
      : "r"(a1), "r"(a3), "r"(a5), "r"(a7), "r"(b));
}

// ---- truncated rows for the squaring: the multiplicand's low limbs are zero, their products are not issued ----
// x[2..7] += (a2, a4, a6) * b at columns 2.. (the lower even limbs of the multiplicand are zero)
B2_D void mad_even_z1(uint32_t* x, uint32_t& top, uint32_t a2, uint32_t a4, uint32_t a6, uint32_t b) {
  asm("mad.lo.cc.u32  %0, %7, %10, %0;\n\t"
      "madc.hi.cc.u32 %1, %7, %10, %1;\n\t"
      "madc.lo.cc.u32 %2, %8, %10, %2;\n\t"
      "madc.hi.cc.u32 %3, %8, %10, %3;\n\t"
      "madc.lo.cc.u32 %4, %9, %10, %4;\n\t"
      "madc.hi.cc.u32 %5, %9, %10, %5;\n\t"
      "addc.u32       %6, %6, 0;"
      : "+r"(x[2]), "+r"(x[3]), "+r"(x[4]), "+r"(x[5]), "+r"(x[6]), "+r"(x[7]), "+r"(top)
      : "r"(a2), "r"(a4), "r"(a6), "r"(b));
}
// x[4..7] += (a4, a6) * b at columns 4.. (the lower even limbs of the multiplicand are zero)
B2_D void mad_even_z2(uint32_t* x, uint32_t& top, uint32_t a4, uint32_t a6, uint32_t b) {
  asm("mad.lo.cc.u32  %0, %5, %7, %0;\n\t"
      "madc.hi.cc.u32 %1, %5, %7, %1;\n\t"
      "madc.lo.cc.u32 %2, %6, %7, %2;\n\t"
      "madc.hi.cc.u32 %3, %6, %7, %3;\n\t"
      "addc.u32       %4, %4, 0;"
      : "+r"(x[4]), "+r"(x[5]), "+r"(x[6]), "+r"(x[7]), "+r"(top)
      : "r"(a4), "r"(a6), "r"(b));
}
// x[6..7] += (a6) * b at columns 6.. (the lower even limbs of the multiplicand are zero)
B2_D void mad_even_z3(uint32_t* x, uint32_t& top, uint32_t a6, uint32_t b) {
  asm("mad.lo.cc.u32  %0, %3, %4, %0;\n\t"
      "madc.hi.cc.u32 %1, %3, %4, %1;\n\t"
      "addc.u32       %2, %2, 0;"
      : "+r"(x[6]), "+r"(x[7]), "+r"(top)
      : "r"(a6), "r"(b));
}
B2_D void shift_mad_odd_z1(uint32_t* e, uint32_t& x0, uint32_t a3, uint32_t a5, uint32_t a7, uint32_t b) {
  asm("add.cc.u32     %8, %8, %1;\n\t"
      "addc.cc.u32    %0, %2, 0;\n\t"
      "addc.cc.u32    %1, %3, 0;\n\t"
      "madc.lo.cc.u32 %2, %9, %12, %4;\n\t"
      "madc.hi.cc.u32 %3, %9, %12, %5;\n\t"
      "madc.lo.cc.u32 %4, %10, %12, %6;\n\t"
      "madc.hi.cc.u32 %5, %10, %12, %7;\n\t"
      "madc.lo.cc.u32 %6, %11, %12, 0;\n\t"
      "madc.hi.u32    %7, %11, %12, 0;"
      : "+r"(e[0]), "+r"(e[1]), "+r"(e[2]), "+r"(e[3]), "+r"(e[4]), "+r"(e[5]), "+r"(e[6]), "+r"(e[7]), "+r"(x0)
      : "r"(a3), "r"(a5), "r"(a7), "r"(b));
}
B2_D void shift_mad_odd_z2(uint32_t* e, uint32_t& x0, uint32_t a5, uint32_t a7, uint32_t b) {
  asm("add.cc.u32     %8, %8, %1;\n\t"
      "addc.cc.u32    %0, %2, 0;\n\t"
      "addc.cc.u32    %1, %3, 0;\n\t"
      "addc.cc.u32    %2, %4, 0;\n\t"
      "addc.cc.u32    %3, %5, 0;\n\t"
      "madc.lo.cc.u32 %4, %9, %11, %6;\n\t"
      "madc.hi.cc.u32 %5, %9, %11, %7;\n\t"
      "madc.lo.cc.u32 %6, %10, %11, 0;\n\t"
      "madc.hi.u32    %7, %10, %11, 0;"
      : "+r"(e[0]), "+r"(e[1]), "+r"(e[2]), "+r"(e[3]), "+r"(e[4]), "+r"(e[5]), "+r"(e[6]), "+r"(e[7]), "+r"(x0)
      : "r"(a5), "r"(a7), "r"(b));
}
B2_D void shift_mad_odd_z3(uint32_t* e, uint32_t& x0, uint32_t a7, uint32_t b) {
  asm("add.cc.u32     %8, %8, %1;\n\t"
      "addc.cc.u32    %0, %2, 0;\n\t"
      "addc.cc.u32    %1, %3, 0;\n\t"
      "addc.cc.u32    %2, %4, 0;\n\t"
      "addc.cc.u32    %3, %5, 0;\n\t"
      "addc.cc.u32    %4, %6, 0;\n\t"
      "addc.cc.u32    %5, %7, 0;\n\t"
      "madc.lo.cc.u32 %6, %9, %10, 0;\n\t"
      "madc.hi.u32    %7, %9, %10, 0;"
      : "+r"(e[0]), "+r"(e[1]), "+r"(e[2]), "+r"(e[3]), "+r"(e[4]), "+r"(e[5]), "+r"(e[6]), "+r"(e[7]), "+r"(x0)
      : "r"(a7), "r"(b));
}

B2_D void mul_even(uint32_t* x, uint32_t a0, uint32_t a2, uint32_t a4, uint32_t a6, uint32_t b) {
  asm("mul.lo.u32 %0, %8,  %12;\n\t mul.hi.u32 %1, %8,  %12;\n\t"
      "mul.lo.u32 %2, %9,  %12;\n\t mul.hi.u32 %3, %9,  %12;\n\t"
      "mul.lo.u32 %4, %10, %12;\n\t mul.hi.u32 %5, %10, %12;\n\t"
      "mul.lo.u32 %6, %11, %12;\n\t mul.hi.u32 %7, %11, %12;"
      : "=r"(x[0]), "=r"(x[1]), "=r"(x[2]), "=r"(x[3]), "=r"(x[4]), "=r"(x[5]), "=r"(x[6]), "=r"(x[7])
      : "r"(a0), "r"(a2), "r"(a4), "r"(a6), "r"(b));
}

// r = a + b (8 limbs), returns nothing: callers guarantee no overflow past 2^256
B2_D void add8(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  asm("add.cc.u32  %0, %8,  %16;\n\t addc.cc.u32 %1, %9,  %17;\n\t addc.cc.u32 %2, %10, %18;\n\t addc.cc.u32 %3, %11, %19;\n\t"
      "addc.cc.u32 %4, %12, %20;\n\t addc.cc.u32 %5, %13, %21;\n\t addc.cc.u32 %6, %14, %22;\n\t addc.u32    %7, %15, %23;"
      : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]),
        "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]), "r"(b[4]), "r"(b[5]), "r"(b[6]), "r"(b[7]));
}
// r = a - b (8 limbs); returns the borrow (0 or 0xffffffff)
B2_D uint32_t sub8(uint32_t* r, const uint32_t* a, const uint32_t* b) {
  uint32_t borrow;
  asm("sub.cc.u32  %0, %9,  %17;\n\t subc.cc.u32 %1, %10, %18;\n\t subc.cc.u32 %2, %11, %19;\n\t subc.cc.u32 %3, %12, %20;\n\t"
      "subc.cc.u32 %4, %13, %21;\n\t subc.cc.u32 %5, %14, %22;\n\t subc.cc.u32 %6, %15, %23;\n\t subc.cc.u32 %7, %16, %24;\n\t"
      "subc.u32    %8, 0, 0;"
      : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]), "=r"(r[4]), "=r"(r[5]), "=r"(r[6]), "=r"(r[7]), "=r"(borrow)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(a[4]), "r"(a[5]), "r"(a[6]), "r"(a[7]),
        "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]), "r"(b[4]), "r"(b[5]), "r"(b[6]), "r"(b[7]));
  return borrow;
}

}  // namespace detail

// ------------------------------------------------------------------------------------------------
template <class Cfg>
struct Fe {
  uint32_t v[8];

  static B2_HD Fe zero() { Fe r; for (int i = 0; i < 8; ++i) r.v[i] = 0; return r; }
  static B2_HD Fe one() { Fe r; for (int i = 0; i < 8; ++i) r.v[i] = Cfg::r1(i); return r; }
  static B2_HD Fe rsquared() { Fe r; for (int i = 0; i < 8; ++i) r.v[i] = Cfg::r2(i); return r; }
  static B2_HD Fe modulus() { Fe r; for (int i = 0; i < 8; ++i) r.v[i] = Cfg::mod(i); return r; }

  B2_HD bool is_zero() const {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) o |= v[i];
    return o == 0;
  }
  B2_HD bool operator==(const Fe& b) const {
    uint32_t o = 0;
#pragma unroll
    for (int i = 0; i < 8; ++i) o |= v[i] ^ b.v[i];
    return o == 0;
  }
  B2_HD bool operator!=(const Fe& b) const { return !(*this == b); }

  // ---- device arithmetic; all values fully reduced: 0 <= v < p ----
  static B2_D Fe reduce_once(const Fe& a) {  // a < 2p  ->  a mod p
    Fe m = modulus(), t;
    uint32_t borrow = detail::sub8(t.v, a.v, m.v);
    Fe r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.v[i] = borrow ? a.v[i] : t.v[i];
    return r;
  }
  static B2_D Fe add(const Fe& a, const Fe& b) {
    Fe s; detail::add8(s.v, a.v, b.v);  // < 2p < 2^255
    return reduce_once(s);
  }
  static B2_D Fe sub(const Fe& a, const Fe& b) {
    Fe d; uint32_t borrow = detail::sub8(d.v, a.v, b.v);
    Fe m;
#pragma unroll
    for (int i = 0; i < 8; ++i) m.v[i] = Cfg::mod(i) & borrow;
    Fe r; detail::add8(r.v, d.v, m.v);
    return r;
  }
  static B2_D Fe dbl(const Fe& a) { return add(a, a); }
  static B2_D Fe neg(const Fe& a) {
    Fe m = modulus(), r; detail::sub8(r.v, m.v, a.v);
    uint32_t nz = a.is_zero() ? 0u : 0xffffffffu;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.v[i] &= nz;
    return r;
  }

  // Montgomery product a*b/2^256 mod p.  Inputs < 2p  =>  before the final subtraction the value is
  // < 4p^2/2^256 + p < 2p (4p < 2^256), so one conditional subtraction canonicalises it, and inside
  // the loop every running total stays below 2^288 (nine 32-bit columns), which is what lets
  // mad_odd / shift_mad_odd end their chains without a carry out.
  static B2_D Fe mul(const Fe& a, const Fe& b) {
    uint32_t ev[8], od[8];
    uint32_t m;
    // round 0
    detail::mul_even(ev, a.v[0], a.v[2], a.v[4], a.v[6], b.v[0]);
    detail::mul_even(od, a.v[1], a.v[3], a.v[5], a.v[7], b.v[0]);
    m = ev[0] * Cfg::INV;
    detail::mad_odd(od, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
    detail::mad_even(ev, od[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
#pragma unroll
    for (int i = 1; i < 8; i += 2) {
      // odd round: `od` is now column-0 aligned, `ev` becomes the odd accumulator
      detail::shift_mad_odd(ev, od[0], a.v[1], a.v[3], a.v[5], a.v[7], b.v[i]);
      detail::mad_even(od, ev[7], a.v[0], a.v[2], a.v[4], a.v[6], b.v[i]);
      m = od[0] * Cfg::INV;
      detail::mad_odd(ev, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
      detail::mad_even(od, ev[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
      if (i + 1 < 8) {
        // even round: roles back
        detail::shift_mad_odd(od, ev[0], a.v[1], a.v[3], a.v[5], a.v[7], b.v[i + 1]);
        detail::mad_even(ev, od[7], a.v[0], a.v[2], a.v[4], a.v[6], b.v[i + 1]);
        m = ev[0] * Cfg::INV;
        detail::mad_odd(od, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
        detail::mad_even(ev, od[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
      }
    }
    // after round 7: `od` is the column-0 aligned accumulator with od[0] == 0, `ev` is column-1 aligned.
    // value / 2^32 = (od >> 32) + ev
    Fe r;
    asm("add.cc.u32  %0, %8,  %16;\n\t addc.cc.u32 %1, %9,  %17;\n\t addc.cc.u32 %2, %10, %18;\n\t addc.cc.u32 %3, %11, %19;\n\t"
        "addc.cc.u32 %4, %12, %20;\n\t addc.cc.u32 %5, %13, %21;\n\t addc.cc.u32 %6, %14, %22;\n\t addc.u32    %7, %15, 0;"
        : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]), "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7])
        : "r"(ev[0]), "r"(ev[1]), "r"(ev[2]), "r"(ev[3]), "r"(ev[4]), "r"(ev[5]), "r"(ev[6]), "r"(ev[7]),
          "r"(od[1]), "r"(od[2]), "r"(od[3]), "r"(od[4]), "r"(od[5]), "r"(od[6]), "r"(od[7]));
    return reduce_once(r);
  }
  // Montgomery square: the same rounds as mul(a, a) with the symmetric products issued once.  Row i multiplies a_i
  // by the vector (0, .., 0, a_i, 2*(a >> 32(i+1))): its limbs are a_i, then d_{i+1} with bit 0 cleared (that bit
  // is a_i's top bit, which belongs to the part not doubled), then d_j -- d = 2a as limbs (a < 2^254, nothing
  // leaves limb 7).  36 wide multiply-adds instead of 64 on the product side; the reduction side is unchanged.
  // Every partial sum is below the full square, and one row is < 2^32 * 2^257, so mul's nine-column bound holds.
  // Limb-exact Python model of this schedule: tools/field_sqr_model.py; the asm itself is executed in simulation by tools/field_asm_sim.py (tests/test_field_asm_model.py).
  static B2_D Fe sqr(const Fe& a) {
    uint32_t d1 = __funnelshift_l(a.v[0], a.v[1], 1), d2 = __funnelshift_l(a.v[1], a.v[2], 1), d3 = __funnelshift_l(a.v[2], a.v[3], 1),
             d4 = __funnelshift_l(a.v[3], a.v[4], 1), d5 = __funnelshift_l(a.v[4], a.v[5], 1), d6 = __funnelshift_l(a.v[5], a.v[6], 1),
             d7 = __funnelshift_l(a.v[6], a.v[7], 1);
    uint32_t ev[8], od[8], m;
    // round 0: (a0, d1', d2, .., d7) * a0
    detail::mul_even(ev, a.v[0], d2, d4, d6, a.v[0]);
    detail::mul_even(od, d1 & ~1u, d3, d5, d7, a.v[0]);
    m = ev[0] * Cfg::INV;
    detail::mad_odd(od, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
    detail::mad_even(ev, od[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
    // round 1: (0, a1, d2', d3, .., d7) * a1
    detail::shift_mad_odd(ev, od[0], a.v[1], d3, d5, d7, a.v[1]);
    detail::mad_even_z1(od, ev[7], d2 & ~1u, d4, d6, a.v[1]);
    m = od[0] * Cfg::INV;
    detail::mad_odd(ev, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
    detail::mad_even(od, ev[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
    // round 2: (0, 0, a2, d3', d4, .., d7) * a2
    detail::shift_mad_odd_z1(od, ev[0], d3 & ~1u, d5, d7, a.v[2]);
    detail::mad_even_z1(ev, od[7], a.v[2], d4, d6, a.v[2]);
    m = ev[0] * Cfg::INV;
    detail::mad_odd(od, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
    detail::mad_even(ev, od[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
    // round 3: (0, 0, 0, a3, d4', d5, d6, d7) * a3
    detail::shift_mad_odd_z1(ev, od[0], a.v[3], d5, d7, a.v[3]);
    detail::mad_even_z2(od, ev[7], d4 & ~1u, d6, a.v[3]);
    m = od[0] * Cfg::INV;
    detail::mad_odd(ev, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
    detail::mad_even(od, ev[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
    // round 4: (.., a4, d5', d6, d7) * a4
    detail::shift_mad_odd_z2(od, ev[0], d5 & ~1u, d7, a.v[4]);
    detail::mad_even_z2(ev, od[7], a.v[4], d6, a.v[4]);
    m = ev[0] * Cfg::INV;
    detail::mad_odd(od, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
    detail::mad_even(ev, od[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
    // round 5: (.., a5, d6', d7) * a5
    detail::shift_mad_odd_z2(ev, od[0], a.v[5], d7, a.v[5]);
    detail::mad_even_z3(od, ev[7], d6 & ~1u, a.v[5]);
    m = od[0] * Cfg::INV;
    detail::mad_odd(ev, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
    detail::mad_even(od, ev[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
    // round 6: (.., a6, d7') * a6
    detail::shift_mad_odd_z3(od, ev[0], d7 & ~1u, a.v[6]);
    detail::mad_even_z3(ev, od[7], a.v[6], a.v[6]);
    m = ev[0] * Cfg::INV;
    detail::mad_odd(od, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
    detail::mad_even(ev, od[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
    // round 7: (.., a7) * a7 -- no even limb left
    detail::shift_mad_odd_z3(ev, od[0], a.v[7], a.v[7]);
    m = od[0] * Cfg::INV;
    detail::mad_odd(ev, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
    detail::mad_even(od, ev[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
    Fe r;
    asm("add.cc.u32  %0, %8,  %16;\n\t addc.cc.u32 %1, %9,  %17;\n\t addc.cc.u32 %2, %10, %18;\n\t addc.cc.u32 %3, %11, %19;\n\t"
        "addc.cc.u32 %4, %12, %20;\n\t addc.cc.u32 %5, %13, %21;\n\t addc.cc.u32 %6, %14, %22;\n\t addc.u32    %7, %15, 0;"
        : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]), "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7])
        : "r"(ev[0]), "r"(ev[1]), "r"(ev[2]), "r"(ev[3]), "r"(ev[4]), "r"(ev[5]), "r"(ev[6]), "r"(ev[7]),
          "r"(od[1]), "r"(od[2]), "r"(od[3]), "r"(od[4]), "r"(od[5]), "r"(od[6]), "r"(od[7]));
    return reduce_once(r);
  }

  // a*b + c*d (Montgomery), ONE reduction for the two products: 24 wide multiply-adds per round instead of
  // 2 x 16.  Bound: with all inputs < p the running total stays below 2^256 + 2*2^286 + 2^286 < 2^288 (nine
  // columns, as in mul) and the result is < 2p^2/2^256 + p < 1.4p, so one conditional subtraction finishes it.
  // The curve formulas use it for Y3 = R*(Q - X3) - Y1*PPP  (c = p - Y1).
  static B2_D Fe mul2_add(const Fe& a, const Fe& b, const Fe& c, const Fe& d) {
    uint32_t ev[8], od[8];
    uint32_t m;
    detail::mul_even(ev, a.v[0], a.v[2], a.v[4], a.v[6], b.v[0]);
    detail::mul_even(od, a.v[1], a.v[3], a.v[5], a.v[7], b.v[0]);
    detail::mad_odd(od, c.v[1], c.v[3], c.v[5], c.v[7], d.v[0]);
    detail::mad_even(ev, od[7], c.v[0], c.v[2], c.v[4], c.v[6], d.v[0]);
    m = ev[0] * Cfg::INV;
    detail::mad_odd(od, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
    detail::mad_even(ev, od[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
#pragma unroll
    for (int i = 1; i < 8; i += 2) {
      detail::shift_mad_odd(ev, od[0], a.v[1], a.v[3], a.v[5], a.v[7], b.v[i]);
      detail::mad_even(od, ev[7], a.v[0], a.v[2], a.v[4], a.v[6], b.v[i]);
      detail::mad_odd(ev, c.v[1], c.v[3], c.v[5], c.v[7], d.v[i]);
      detail::mad_even(od, ev[7], c.v[0], c.v[2], c.v[4], c.v[6], d.v[i]);
      m = od[0] * Cfg::INV;
      detail::mad_odd(ev, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
      detail::mad_even(od, ev[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
      if (i + 1 < 8) {
        detail::shift_mad_odd(od, ev[0], a.v[1], a.v[3], a.v[5], a.v[7], b.v[i + 1]);
        detail::mad_even(ev, od[7], a.v[0], a.v[2], a.v[4], a.v[6], b.v[i + 1]);
        detail::mad_odd(od, c.v[1], c.v[3], c.v[5], c.v[7], d.v[i + 1]);
        detail::mad_even(ev, od[7], c.v[0], c.v[2], c.v[4], c.v[6], d.v[i + 1]);
        m = ev[0] * Cfg::INV;
        detail::mad_odd(od, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
        detail::mad_even(ev, od[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
      }
    }
    Fe r;
    asm("add.cc.u32  %0, %8,  %16;\n\t addc.cc.u32 %1, %9,  %17;\n\t addc.cc.u32 %2, %10, %18;\n\t addc.cc.u32 %3, %11, %19;\n\t"
        "addc.cc.u32 %4, %12, %20;\n\t addc.cc.u32 %5, %13, %21;\n\t addc.cc.u32 %6, %14, %22;\n\t addc.u32    %7, %15, 0;"
        : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]), "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7])
        : "r"(ev[0]), "r"(ev[1]), "r"(ev[2]), "r"(ev[3]), "r"(ev[4]), "r"(ev[5]), "r"(ev[6]), "r"(ev[7]),
          "r"(od[1]), "r"(od[2]), "r"(od[3]), "r"(od[4]), "r"(od[5]), "r"(od[6]), "r"(od[7]));
    return reduce_once(r);
  }
  // a*b + c*d + e*f + g*h (Montgomery), ONE reduction for the four products: 40 wide multiply-adds per round instead
  // of 4 x 16.  Bound (both moduli are 0.756 * 2^254): a round adds at most 4 * p * 2^32 + p * 2^32 = 0.945 * 2^288 to a
  // running total below 2^256, so the nine columns still hold it, and the result is < 4p^2/2^256 + p = 1.76p: one
  // conditional subtraction.  Checked at the worst case ((p-1)^2 four times) by tools/field_sqr_model.py.
  // Fq2's a*b - c*d uses it for each of its two components.
  static B2_D Fe mul4_add(const Fe& a, const Fe& b, const Fe& c, const Fe& d, const Fe& e, const Fe& f, const Fe& g, const Fe& h) {
    const Fe* const x[4] = {&a, &c, &e, &g};
    const Fe* const y[4] = {&b, &d, &f, &h};
    uint32_t ev[8], od[8];
    uint32_t m;
    detail::mul_even(ev, a.v[0], a.v[2], a.v[4], a.v[6], b.v[0]);
    detail::mul_even(od, a.v[1], a.v[3], a.v[5], a.v[7], b.v[0]);
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      detail::mad_odd(od, x[k]->v[1], x[k]->v[3], x[k]->v[5], x[k]->v[7], y[k]->v[0]);
      detail::mad_even(ev, od[7], x[k]->v[0], x[k]->v[2], x[k]->v[4], x[k]->v[6], y[k]->v[0]);
    }
    m = ev[0] * Cfg::INV;
    detail::mad_odd(od, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
    detail::mad_even(ev, od[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
#pragma unroll
    for (int i = 1; i < 8; i += 2) {
      detail::shift_mad_odd(ev, od[0], a.v[1], a.v[3], a.v[5], a.v[7], b.v[i]);
      detail::mad_even(od, ev[7], a.v[0], a.v[2], a.v[4], a.v[6], b.v[i]);
#pragma unroll
      for (int k = 1; k < 4; ++k) {
        detail::mad_odd(ev, x[k]->v[1], x[k]->v[3], x[k]->v[5], x[k]->v[7], y[k]->v[i]);
        detail::mad_even(od, ev[7], x[k]->v[0], x[k]->v[2], x[k]->v[4], x[k]->v[6], y[k]->v[i]);
      }
      m = od[0] * Cfg::INV;
      detail::mad_odd(ev, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
      detail::mad_even(od, ev[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
      if (i + 1 < 8) {
        detail::shift_mad_odd(od, ev[0], a.v[1], a.v[3], a.v[5], a.v[7], b.v[i + 1]);
        detail::mad_even(ev, od[7], a.v[0], a.v[2], a.v[4], a.v[6], b.v[i + 1]);
#pragma unroll
        for (int k = 1; k < 4; ++k) {
          detail::mad_odd(od, x[k]->v[1], x[k]->v[3], x[k]->v[5], x[k]->v[7], y[k]->v[i + 1]);
          detail::mad_even(ev, od[7], x[k]->v[0], x[k]->v[2], x[k]->v[4], x[k]->v[6], y[k]->v[i + 1]);
        }
        m = ev[0] * Cfg::INV;
        detail::mad_odd(od, Cfg::mod(1), Cfg::mod(3), Cfg::mod(5), Cfg::mod(7), m);
        detail::mad_even(ev, od[7], Cfg::mod(0), Cfg::mod(2), Cfg::mod(4), Cfg::mod(6), m);
      }
    }
    Fe r;
    asm("add.cc.u32  %0, %8,  %16;\n\t addc.cc.u32 %1, %9,  %17;\n\t addc.cc.u32 %2, %10, %18;\n\t addc.cc.u32 %3, %11, %19;\n\t"
        "addc.cc.u32 %4, %12, %20;\n\t addc.cc.u32 %5, %13, %21;\n\t addc.cc.u32 %6, %14, %22;\n\t addc.u32    %7, %15, 0;"
        : "=r"(r.v[0]), "=r"(r.v[1]), "=r"(r.v[2]), "=r"(r.v[3]), "=r"(r.v[4]), "=r"(r.v[5]), "=r"(r.v[6]), "=r"(r.v[7])
        : "r"(ev[0]), "r"(ev[1]), "r"(ev[2]), "r"(ev[3]), "r"(ev[4]), "r"(ev[5]), "r"(ev[6]), "r"(ev[7]),
          "r"(od[1]), "r"(od[2]), "r"(od[3]), "r"(od[4]), "r"(od[5]), "r"(od[6]), "r"(od[7]));
    return reduce_once(r);
  }
  // a*b - c*d
  static B2_D Fe mul2_sub(const Fe& a, const Fe& b, const Fe& c, const Fe& d) { return mul2_add(a, b, neg(c), d); }

  static B2_D Fe to_mont(const Fe& canonical) { return mul(canonical, rsquared()); }
  static B2_D Fe from_mont(const Fe& a) {
    Fe o = zero(); o.v[0] = 1; return mul(a, o);
  }
  // a^e, e = 256-bit little-endian limbs (square-and-multiply, MSB first)
  static B2_D Fe pow(const Fe& a, const uint32_t* e) {
    Fe acc = one();
    for (int i = 255; i >= 0; --i) {
      acc = sqr(acc);
      if ((e[i >> 5] >> (i & 31)) & 1) acc = mul(acc, a);
    }
    return acc;
  }
  static B2_D Fe inv(const Fe& a) {  // Fermat: a^(p-2); inv(0) = 0
    uint32_t e[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) e[i] = Cfg::mod(i);
    e[0] -= 2;  // both moduli end in ...01 / ...47: no borrow
    return pow(a, e);
  }
};

typedef Fe<FqCfg> Fq;
typedef Fe<FrCfg> Fr;

// Fq2 = Fq[u]/(u^2+1); c0 = real, c1 = imaginary.
struct Fq2 {
  Fq c0, c1;
  static B2_D Fq2 zero() { return {Fq::zero(), Fq::zero()}; }
  static B2_D Fq2 one() { return {Fq::one(), Fq::zero()}; }
  B2_D bool is_zero() const { return c0.is_zero() && c1.is_zero(); }
  B2_D bool operator==(const Fq2& b) const { return c0 == b.c0 && c1 == b.c1; }
  B2_D bool operator!=(const Fq2& b) const { return !(*this == b); }
  static B2_D Fq2 add(const Fq2& a, const Fq2& b) { return {Fq::add(a.c0, b.c0), Fq::add(a.c1, b.c1)}; }
  static B2_D Fq2 sub(const Fq2& a, const Fq2& b) { return {Fq::sub(a.c0, b.c0), Fq::sub(a.c1, b.c1)}; }
  static B2_D Fq2 dbl(const Fq2& a) { return {Fq::dbl(a.c0), Fq::dbl(a.c1)}; }
  static B2_D Fq2 neg(const Fq2& a) { return {Fq::neg(a.c0), Fq::neg(a.c1)}; }
  // Schoolbook with ONE reduction per component: c0 = a0 b0 + (p - a1) b1, c1 = a0 b1 + a1 b0 -- 2 x 200 multiply
  // instructions and one negation.  Karatsuba (3 x 136 and five additions/subtractions with their temporaries) was
  // the first version and slower: the register pressure of the temporaries cost more than the 8 multiply instructions saved.
  static B2_D Fq2 mul(const Fq2& a, const Fq2& b) {
    return {Fq::mul2_add(a.c0, b.c0, Fq::neg(a.c1), b.c1), Fq::mul2_add(a.c0, b.c1, a.c1, b.c0)};
  }
  static B2_D Fq2 sqr(const Fq2& a) {  // (c0+c1)(c0-c1), 2 c0 c1
    Fq s = Fq::add(a.c0, a.c1), d = Fq::sub(a.c0, a.c1), m = Fq::mul(a.c0, a.c1);
    return {Fq::mul(s, d), Fq::dbl(m)};
  }
  // a*b - c*d over Fq2: each component is a sum of FOUR base-field products under one reduction (Fq::mul4_add):
  //   re = a0 b0 - a1 b1 - c0 d0 + c1 d1        im = a0 b1 + a1 b0 - c0 d1 - c1 d0
  static B2_D Fq2 mul2_sub(const Fq2& a, const Fq2& b, const Fq2& c, const Fq2& d) {
#ifdef B200ZK_FQ2_NO_MUL4
    return sub(mul(a, b), mul(c, d));
#else
    const Fq na1 = Fq::neg(a.c1), nc0 = Fq::neg(c.c0), nc1 = Fq::neg(c.c1);
    return {Fq::mul4_add(a.c0, b.c0, na1, b.c1, nc0, d.c0, c.c1, d.c1), Fq::mul4_add(a.c0, b.c1, a.c1, b.c0, nc0, d.c1, nc1, d.c0)};
#endif
  }
  static B2_D Fq2 inv(const Fq2& a) {
    Fq d = Fq::inv(Fq::add(Fq::sqr(a.c0), Fq::sqr(a.c1)));
    return {Fq::mul(a.c0, d), Fq::neg(Fq::mul(a.c1, d))};
  }
};

}  // namespace b200zk
