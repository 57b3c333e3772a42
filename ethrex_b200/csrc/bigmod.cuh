// bigmod.cuh -- multi-precision arithmetic modulo a runtime modulus for sm_90a: the MODEXP precompile (modexp.cu).
//
// A number of N 32-bit limbs (little-endian) is spread over the TPI threads of one group inside a warp, kLimbs = N / TPI
// = 8 limbs per thread (lane l holds limbs l*8 .. l*8+7), the same register budget per thread as the BN254 field core.
// modexp.cu instantiates N = 8, 32, 64, 128, 256 with TPI = 1, 4, 8, 16, 32.  Several groups share a warp when TPI < 32,
// so every shuffle and ballot names the group's own lanes only (Group::mask) and groups may diverge freely; nothing here
// synchronises more than a group, and TPI = 1 takes no shuffle at all.
//
// Montgomery product (CIOS, R = 2^(32N)).  Round i (i = 0 .. N-1) broadcasts b_i from the lane that owns it, adds a*b_i
// to the accumulator t row by row (one 64-bit multiply-add per limb: t + a*b + c < 2^64), broadcasts q = t_0 m' from
// lane 0, adds q*m the same way, and shifts t down one limb: each lane takes its upper neighbour's limb 0.  The carry
// out of a lane's row is not passed on at once: each lane keeps it in a pending word p that stands at the position of
// its upper neighbour's limb 0, and the shift folds p into the limb that arrives there (that sum, p + two row carries
// + a limb, is < 2^34, so p stays below 4 after the first round).  So a round costs two shuffles of data (b_i, q) and
// one for the shift, and no carry ever crosses a lane inside the loop.  After the last round the pending words are
// resolved once (each lane adds its lower neighbour's p, leaving a carry of 0 or 1 per lane, which a ballot of
// generate / all-ones-propagate bits resolves across the group in one step: carry-in bits = ((G << 1) + P) ^ P), and
// the result t < 2m is brought below m by a group-wide compare: t - m with the same ballot borrow resolution, kept when
// the top word does not borrow.
//
// Products are valid for a < R, b < m (or the other way round) and any odd m < R; the result is < m.  lo_mul is the
// same loop without the reduction: the limb leaving lane 0 at round i is limb i of a*b mod R (the pending carries
// stand at lane boundaries above it, so it is final), and lane i / 8 keeps it.  It serves the 2^s factor of an even
// modulus (modexp.cu), where arithmetic mod 2^s is arithmetic mod R truncated to s bits at the end.
//
// No division anywhere: m' = -m^-1 mod 2^32 and q^-1 mod R come from Newton iterations, R mod m and R^2 mod m from
// 2 * 32N modular doublings.
#pragma once
#include <cstdint>

#include "field.cuh"  // B2_D

namespace b200zk {
namespace bigmod {

constexpr int kLimbs = 8;  // limbs per thread, every class

// the TPI lanes that share one number: lane = index inside the group, shift = position of the group's bits in a ballot
template <int TPI> struct Group {
  uint32_t mask;
  uint32_t lane;
  uint32_t shift;
  B2_D Group() {
    const uint32_t wl = threadIdx.x & 31;
    lane = wl % TPI;
    shift = wl - lane;
    mask = TPI == 32 ? 0xffffffffu : ((1u << TPI) - 1u) << shift;
  }
  B2_D uint32_t bcast(uint32_t x, uint32_t src) const {
    if constexpr (TPI == 1) return x;
    else return __shfl_sync(mask, x, src, TPI);
  }
  // x of lane + 1; 0 on the top lane
  B2_D uint32_t from_above(uint32_t x) const {
    if constexpr (TPI == 1) return 0;
    else {
      const uint32_t v = __shfl_down_sync(mask, x, 1, TPI);
      return lane == TPI - 1 ? 0 : v;
    }
  }
  // x of lane - 1; 0 on lane 0
  B2_D uint32_t from_below(uint32_t x) const {
    if constexpr (TPI == 1) return 0;
    else {
      const uint32_t v = __shfl_up_sync(mask, x, 1, TPI);
      return lane == 0 ? 0 : v;
    }
  }
  // one bit per lane of the group, lane 0 = bit 0
  B2_D uint64_t ballot(bool pred) const {
    if constexpr (TPI == 1) return pred ? 1u : 0u;
    else return (uint64_t)((__ballot_sync(mask, pred) & mask) >> shift);
  }
  B2_D bool any(bool pred) const { return ballot(pred) != 0; }
};

template <int TPI> struct Num { uint32_t v[kLimbs]; };

template <int TPI> B2_D void set_small(Num<TPI>& a, const Group<TPI>& g, uint32_t x) {
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) a.v[k] = 0;
  if (g.lane == 0) a.v[0] = x;
}

template <int TPI> B2_D bool is_zero(const Num<TPI>& a, const Group<TPI>& g) {
  uint32_t o = 0;
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) o |= a.v[k];
  return !g.any(o != 0);
}

template <int TPI> B2_D bool is_one(const Num<TPI>& a, const Group<TPI>& g) {
  uint32_t o = g.lane == 0 ? a.v[0] ^ 1u : a.v[0];
#pragma unroll
  for (int k = 1; k < kLimbs; ++k) o |= a.v[k];
  return !g.any(o != 0);
}

// the carry (or borrow) into this lane, and out of the top lane, from per-lane generate bits and all-ones (all-zero)
// propagate bits; a lane never both generates and propagates
template <int TPI> B2_D void resolve(const Group<TPI>& g, bool gen, bool prop, uint32_t& cin, uint32_t& cout) {
  const uint64_t G = g.ballot(gen), P = g.ballot(prop);
  const uint64_t C = ((G << 1) + P) ^ P;
  cin = (uint32_t)(C >> g.lane) & 1u;
  cout = (uint32_t)(C >> TPI) & 1u;
}

// a += c within the lane; returns the carry out (0 or 1 for c < 2^32)
template <int TPI> B2_D uint32_t add_word(Num<TPI>& a, uint32_t c) {
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) {
    const uint64_t s = (uint64_t)a.v[k] + c;
    a.v[k] = (uint32_t)s;
    c = (uint32_t)(s >> 32);
  }
  return c;
}

template <int TPI> B2_D uint32_t sub_word(Num<TPI>& a, uint32_t b) {
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) {
    const uint32_t x = a.v[k];
    a.v[k] = x - b;
    b = x < b ? 1u : 0u;
  }
  return b;
}

template <int TPI> B2_D bool all_ones(const Num<TPI>& a) {
  uint32_t x = 0xffffffffu;
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) x &= a.v[k];
  return x == 0xffffffffu;
}

template <int TPI> B2_D bool all_zero(const Num<TPI>& a) {
  uint32_t x = 0;
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) x |= a.v[k];
  return x == 0;
}

// a += b over the group; returns the carry out of the top limb (same on every lane)
template <int TPI> B2_D uint32_t add(Num<TPI>& a, const Num<TPI>& b, const Group<TPI>& g) {
  uint32_t c = 0;
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) {
    const uint64_t s = (uint64_t)a.v[k] + b.v[k] + c;
    a.v[k] = (uint32_t)s;
    c = (uint32_t)(s >> 32);
  }
  uint32_t cin, cout;
  resolve(g, c != 0, all_ones(a), cin, cout);
  add_word(a, cin);
  return cout;
}

// a -= b over the group; returns the borrow out of the top limb
template <int TPI> B2_D uint32_t sub(Num<TPI>& a, const Num<TPI>& b, const Group<TPI>& g) {
  uint32_t br = 0;
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) {
    const uint32_t x = a.v[k], y = b.v[k];
    const uint32_t d = x - y;
    const uint32_t nb = (x < y) | (d < br);
    a.v[k] = d - br;
    br = nb;
  }
  uint32_t bin, bout;
  resolve(g, br != 0, all_zero(a), bin, bout);
  sub_word(a, bin);
  return bout;
}

// t + hi * R, known < 2m, reduced below m (hi is the same on every lane)
template <int TPI> B2_D void cond_sub(Num<TPI>& t, uint32_t hi, const Num<TPI>& m, const Group<TPI>& g) {
  Num<TPI> d = t;
  const uint32_t borrow = sub(d, m, g);
  if (hi || !borrow) t = d;
}

// (a + b) mod m for a, b < m
template <int TPI> B2_D void mod_add(Num<TPI>& a, const Num<TPI>& b, const Num<TPI>& m, const Group<TPI>& g) {
  const uint32_t hi = add(a, b, g);
  cond_sub(a, hi, m, g);
}

// 2a mod m for a < m
template <int TPI> B2_D void mod_dbl(Num<TPI>& a, const Num<TPI>& m, const Group<TPI>& g) {
  const uint32_t below = g.from_below(a.v[kLimbs - 1] >> 31);
  const uint32_t hi = g.bcast(a.v[kLimbs - 1] >> 31, TPI - 1);
#pragma unroll
  for (int k = kLimbs - 1; k > 0; --k) a.v[k] = (a.v[k] << 1) | (a.v[k - 1] >> 31);
  a.v[0] = (a.v[0] << 1) | below;
  cond_sub(a, hi, m, g);
}

// t += a * b (one row); returns the carry out of the lane's top limb
template <int TPI> B2_D uint32_t mad_row(Num<TPI>& t, const Num<TPI>& a, uint32_t b) {
  uint32_t c = 0;
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) {
    const uint64_t s = (uint64_t)a.v[k] * b + t.v[k] + c;
    t.v[k] = (uint32_t)s;
    c = (uint32_t)(s >> 32);
  }
  return c;
}

// t / 2^32, the lane's pending word and this round's row carries folded into the limb arriving from above
template <int TPI> B2_D void shift_down(Num<TPI>& t, uint32_t& p, uint32_t c1, uint32_t c2, const Group<TPI>& g) {
  const uint64_t top = (uint64_t)g.from_above(t.v[0]) + p + c1 + c2;
#pragma unroll
  for (int k = 0; k < kLimbs - 1; ++k) t.v[k] = t.v[k + 1];
  t.v[kLimbs - 1] = (uint32_t)top;
  p = (uint32_t)(top >> 32);
}

// -x^-1 mod 2^32 for odd x (Newton: 3 correct bits, doubled four times)
B2_D uint32_t neg_inv32(uint32_t x) {
  uint32_t y = x;
#pragma unroll
  for (int i = 0; i < 4; ++i) y *= 2u - x * y;
  return 0u - y;
}

// a * b / R mod m; m odd, mp = -m^-1 mod 2^32, a < R and b < m (or the other way round)
template <int TPI> B2_D Num<TPI> mont_mul(const Num<TPI>& a, const Num<TPI>& b, const Num<TPI>& m, uint32_t mp, const Group<TPI>& g) {
  Num<TPI> t;
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) t.v[k] = 0;
  uint32_t p = 0;
  for (uint32_t src = 0; src < TPI; ++src) {
#pragma unroll
    for (int k = 0; k < kLimbs; ++k) {
      const uint32_t bi = g.bcast(b.v[k], src);
      const uint32_t c1 = mad_row(t, a, bi);
      const uint32_t q = g.bcast(t.v[0] * mp, 0);
      const uint32_t c2 = mad_row(t, m, q);
      shift_down(t, p, c1, c2, g);
    }
  }
  // resolve the pending words: each lane takes its lower neighbour's, then one ballot settles the 0/1 carries
  const uint32_t co = add_word(t, g.from_below(p));
  uint32_t cin, cout;
  resolve(g, co != 0, all_ones(t), cin, cout);
  add_word(t, cin);
  cond_sub(t, g.bcast(p, TPI - 1) + cout, m, g);
  return t;
}

// a * b mod R
template <int TPI> B2_D Num<TPI> lo_mul(const Num<TPI>& a, const Num<TPI>& b, const Group<TPI>& g) {
  Num<TPI> t, r;
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) t.v[k] = 0;
  uint32_t p = 0;
  for (uint32_t src = 0; src < TPI; ++src) {
#pragma unroll
    for (int k = 0; k < kLimbs; ++k) {
      const uint32_t bi = g.bcast(b.v[k], src);
      const uint32_t c1 = mad_row(t, a, bi);
      const uint32_t out = g.bcast(t.v[0], 0);
      if (g.lane == src) r.v[k] = out;
      shift_down(t, p, c1, 0u, g);
    }
  }
  return r;
}

// a mod 2^s
template <int TPI> B2_D void truncate_bits(Num<TPI>& a, uint32_t s, const Group<TPI>& g) {
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) {
    const uint32_t bit = 32u * (g.lane * kLimbs + k);
    if (bit >= s) a.v[k] = 0;
    else if (s - bit < 32) a.v[k] &= (1u << (s - bit)) - 1u;
  }
}

// q^-1 mod R for odd q: Newton x <- x (2 - q x), 32 correct bits doubled log2(N) times
template <int TPI> B2_D Num<TPI> inv_mod_r(const Num<TPI>& q, const Group<TPI>& g) {
  Num<TPI> x;
  set_small(x, g, 0u - neg_inv32(g.bcast(q.v[0], 0)));
  for (int bits = 32; bits < 32 * kLimbs * TPI; bits *= 2) {
    Num<TPI> y = lo_mul(q, x, g);
#pragma unroll
    for (int k = 0; k < kLimbs; ++k) y.v[k] = ~y.v[k];  // 2 - y = ~y + 3 mod R
    uint32_t cin, cout;
    const uint32_t co = add_word(y, g.lane == 0 ? 3u : 0u);
    resolve(g, co != 0, all_ones(y), cin, cout);
    add_word(y, cin);
    x = lo_mul(x, y, g);
  }
  return x;
}

}  // namespace bigmod
}  // namespace b200zk
