// modexp.cu -- batched MODEXP on the device: Crypto::modexp of the reference (crates/common/crypto/provider.rs:334-380,
// levm precompile 0x05 at precompiles.rs:559-643), `count` independent items per call with EIP-7823's 1024-byte bound on
// each operand.  The arithmetic is in bigmod.cuh; this file holds the size classes, the kernel and the C entry point.
#include <algorithm>

#include "common.cuh"
#include "bigmod.cuh"

namespace b200zk {
namespace {

using bigmod::Group;
using bigmod::kLimbs;
using bigmod::Num;

constexpr int kModexpThreads = 64;
constexpr int kWindow = 16;  // 4-bit fixed window: 16 table entries per item
constexpr int kClasses = 5;
// modulus size classes: N 32-bit limbs on TPI lanes, 8 limbs per lane (256 .. 8192 bits)
constexpr uint32_t kClassLimbs[kClasses] = {8, 32, 64, 128, 256};
constexpr uint8_t kOverBound = 2;  // status of an item with an operand longer than B200ZK_MODEXP_MAX_BYTES

// one item as the kernel sees it: byte offsets into the upload, leading zero bytes of base, exponent and modulus
// stripped (mod_len >= 1); out_len = the caller's modulus length, the width of the item's output slot
struct ModexpItem {
  uint64_t base, exp, mod, out;
  uint32_t base_len, exp_len, mod_len, out_len;
};

// limbs limb0 .. limb0 + N - 1 of the big-endian byte string p[0 .. len), this lane's eight of them
template <int TPI> B2_D Num<TPI> load_be(const uint8_t* p, uint32_t len, uint32_t limb0, const Group<TPI>& g) {
  Num<TPI> a;
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) {
    const uint32_t gi = limb0 + g.lane * kLimbs + k;
    uint32_t v = 0;
#pragma unroll
    for (int b = 3; b >= 0; --b) {
      const uint32_t idx = 4 * gi + b;
      v = (v << 8) | (idx < len ? p[len - 1 - idx] : 0u);
    }
    a.v[k] = v;
  }
  return a;
}

// window table in shared memory, lane-interleaved: entry w, limb k of lane l at (w * 8 + k) * TPI + l
template <int TPI> B2_D void tab_store(uint32_t* tab, uint32_t w, const Num<TPI>& a, const Group<TPI>& g) {
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) tab[(w * kLimbs + k) * TPI + g.lane] = a.v[k];
}
template <int TPI> B2_D Num<TPI> tab_load(const uint32_t* tab, uint32_t w, const Group<TPI>& g) {
  Num<TPI> a;
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) a.v[k] = tab[(w * kLimbs + k) * TPI + g.lane];
  return a;
}

// base^e under mul (one = its unit), e = the big-endian bytes e[0 .. elen) with e[0] != 0, scanned MSB first in 4-bit
// windows; e = 0 (elen = 0) gives one.  Each lane reads back only the table limbs it wrote.
template <int TPI, class Mul>
B2_D Num<TPI> pow_window(uint32_t* tab, const Num<TPI>& one, const Num<TPI>& base, const uint8_t* e, uint32_t elen, Mul mul,
                         const Group<TPI>& g) {
  if (elen == 0) return one;
  tab_store(tab, 1, base, g);
  Num<TPI> x = base;
  for (uint32_t w = 2; w < kWindow; ++w) {
    x = mul(x, base);
    tab_store(tab, w, x, g);
  }
  bool started = false;
  for (uint32_t i = 0; i < 2 * elen; ++i) {
    const uint32_t byte = e[i >> 1];
    const uint32_t nib = (i & 1) ? byte & 15u : byte >> 4;
    if (started) {
#pragma unroll 1
      for (int j = 0; j < 4; ++j) x = mul(x, x);
    }
    if (nib) {
      const Num<TPI> y = tab_load(tab, nib, g);
      x = started ? mul(x, y) : y;
      started = true;
    }
  }
  return x;
}

// One item per group of TPI lanes.  m = 2^s q with q odd: r_q = b^e mod q on the Montgomery path (skipped when q = 1),
// r_2 = b^e mod 2^s with products mod R truncated to s bits (skipped when s = 0), and the CRT
// x = r_q + q ((r_2 - r_q) q^-1 mod 2^s), which is < m.
template <int N, int TPI>
__global__ void __launch_bounds__(kModexpThreads) modexp_kernel(const uint8_t* __restrict__ data, const ModexpItem* __restrict__ items,
                                                                uint32_t n, uint8_t* __restrict__ out) {
  static_assert(N == kLimbs * TPI, "eight limbs per lane");
  extern __shared__ uint32_t smem[];
  const Group<TPI> g;
  const uint32_t slot = threadIdx.x / TPI;
  const uint32_t idx = blockIdx.x * (kModexpThreads / TPI) + slot;
  if (idx >= n) return;  // the whole group leaves together
  const ModexpItem it = items[idx];
  uint32_t* tab = smem + slot * kWindow * N;
  const uint8_t* e = data + it.exp;

  const Num<TPI> m = load_be(data + it.mod, it.mod_len, 0, g);
  // s = trailing zero bits of m (m != 0): the lowest lane holding a nonzero limb says where
  uint32_t tz = 0xffffffffu;
#pragma unroll
  for (int k = kLimbs - 1; k >= 0; --k)
    if (m.v[k]) tz = 32u * (g.lane * kLimbs + k) + __ffs(m.v[k]) - 1;
  const uint32_t s = g.bcast(tz, __ffsll((long long)g.ballot(tz != 0xffffffffu)) - 1);
  Num<TPI> q = m;
  if (s) {  // q = m >> s through the table's space
#pragma unroll
    for (int k = 0; k < kLimbs; ++k) tab[g.lane * kLimbs + k] = m.v[k];
    __syncwarp(g.mask);
    const uint32_t ls = s / 32, bs = s % 32;
#pragma unroll
    for (int k = 0; k < kLimbs; ++k) {
      const uint32_t src = g.lane * kLimbs + k + ls;
      const uint32_t lo = src < N ? tab[src] : 0u, hi = src + 1 < N ? tab[src + 1] : 0u;
      q.v[k] = bs ? (lo >> bs) | (hi << (32 - bs)) : lo;
    }
    __syncwarp(g.mask);
  }

  Num<TPI> one, rq;
  bigmod::set_small(one, g, 1);
  bigmod::set_small(rq, g, 0);
  if (!bigmod::is_one(q, g)) {
    const uint32_t mp = g.bcast(bigmod::neg_inv32(q.v[0]), 0);
    auto mont = [&](const Num<TPI>& a, const Num<TPI>& b) { return bigmod::mont_mul(a, b, q, mp, g); };
    Num<TPI> r1 = one;  // R mod q, then R^2 mod q, by doublings
    for (uint32_t j = 0; j < 32 * N; ++j) bigmod::mod_dbl(r1, q, g);
    Num<TPI> r2 = r1;
    for (uint32_t j = 0; j < 32 * N; ++j) bigmod::mod_dbl(r2, q, g);
    // b R mod q by Horner over N-limb chunks, top chunk first: acc <- acc R + c (each chunk < R, taken times R^2 / R)
    Num<TPI> bm;
    bigmod::set_small(bm, g, 0);
    const uint32_t chunks = (it.base_len + 4 * N - 1) / (4 * N);
    for (uint32_t c = chunks; c-- > 0;) {
      const Num<TPI> ck = mont(load_be(data + it.base, it.base_len, c * N, g), r2);
      if (c + 1 == chunks) {
        bm = ck;
      } else {
        bm = mont(bm, r2);
        bigmod::mod_add(bm, ck, q, g);
      }
    }
    const Num<TPI> x = pow_window(tab, r1, bm, e, it.exp_len, mont, g);
    rq = mont(x, one);  // out of Montgomery form
  }
  Num<TPI> res = rq;
  if (s) {
    auto lo = [&](const Num<TPI>& a, const Num<TPI>& b) { return bigmod::lo_mul(a, b, g); };
    Num<TPI> r2 = pow_window(tab, one, load_be(data + it.base, it.base_len, 0, g), e, it.exp_len, lo, g);
    bigmod::sub(r2, rq, g);
    bigmod::truncate_bits(r2, s, g);
    Num<TPI> h = bigmod::lo_mul(r2, bigmod::inv_mod_r(q, g), g);
    bigmod::truncate_bits(h, s, g);
    res = bigmod::lo_mul(q, h, g);  // q h < q 2^s = m < R: the low half is the whole product
    bigmod::add(res, rq, g);
  }

  // the low mod_len bytes of the output slot, big-endian; the bytes above them were zeroed before the launch
  uint8_t* o = out + it.out + it.out_len - 1;
#pragma unroll
  for (int k = 0; k < kLimbs; ++k) {
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const uint32_t i = 4 * (g.lane * kLimbs + k) + b;
      if (i < it.mod_len) *(o - i) = (uint8_t)(res.v[k] >> (8 * b));
    }
  }
}

template <int N>
int launch_class(b200zk_ctx* ctx, cudaStream_t st, const uint8_t* din, const ModexpItem* ditems, uint32_t n, uint8_t* dout) {
  constexpr int TPI = N / kLimbs;
  constexpr int per_block = kModexpThreads / TPI;
  constexpr size_t smem = (size_t)per_block * kWindow * N * sizeof(uint32_t);  // 32 KiB in every class
  B2_LAUNCH(ctx, (modexp_kernel<N, TPI>), (n + per_block - 1) / per_block, kModexpThreads, smem, st, din, ditems, n, dout);
  return B200ZK_OK;
}

int class_of(uint32_t mod_bytes) {
  const uint32_t limbs = (mod_bytes + 3) / 4;
  int c = 0;
  while (kClassLimbs[c] < limbs) ++c;
  return c;
}

// leading zero bytes of p[0 .. len)
uint32_t leading_zeros(const uint8_t* p, uint32_t len) {
  uint32_t z = 0;
  while (z < len && !p[z]) ++z;
  return z;
}

}  // namespace
}  // namespace b200zk

using namespace b200zk;

extern "C" {

int b200zk_modexp_batch(b200zk_ctx* ctx, const uint8_t* data, const uint32_t* lens, size_t count, uint8_t* out, uint8_t* status) {
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  if (count && (!data || !lens || !out || !status)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "modexp_batch: null argument");
  NvtxRange nvtx("b200zk:modexp_batch");
  DeviceGuard guard(ctx);
  if (!count) return B200ZK_OK;
  if (count > UINT32_MAX) return fail(ctx, B200ZK_ERR_INVALID_ARG, "modexp_batch: more than 2^32 - 1 items");
  // offsets, statuses and the kernel's items per class on the host: one pass over the lengths and the leading bytes
  std::vector<ModexpItem> cls[kClasses];
  size_t in_total = 0, out_total = 0;
  for (size_t i = 0; i < count; ++i) {
    const uint32_t bl = lens[3 * i], el = lens[3 * i + 1], ml = lens[3 * i + 2];
    const size_t b = in_total;
    size_t e, m, end, oend;
    if (__builtin_add_overflow(b, (size_t)bl, &e) || __builtin_add_overflow(e, (size_t)el, &m) ||
        __builtin_add_overflow(m, (size_t)ml, &end) || __builtin_add_overflow(out_total, (size_t)ml, &oend))
      return fail(ctx, B200ZK_ERR_INVALID_ARG, "modexp_batch: operand lengths overflow size_t");
    const size_t o = out_total;
    in_total = end;
    out_total = oend;
    const bool over = bl > B200ZK_MODEXP_MAX_BYTES || el > B200ZK_MODEXP_MAX_BYTES || ml > B200ZK_MODEXP_MAX_BYTES;
    status[i] = over ? kOverBound : B200ZK_OK;
    if (over) continue;
    const uint32_t mz = leading_zeros(data + m, ml);
    if (mz == ml) continue;  // m = 0: the output stays zero
    const uint32_t bz = leading_zeros(data + b, bl), ez = leading_zeros(data + e, el);
    cls[class_of(ml - mz)].push_back({b + bz, e + ez, m + mz, o, bl - bz, el - ez, ml - mz, ml});
  }
  // longest exponents first inside a class, so the long chains start first and warp-mates finish together
  std::vector<ModexpItem> items;
  uint32_t first[kClasses + 1] = {0};
  for (int c = 0; c < kClasses; ++c) {
    std::stable_sort(cls[c].begin(), cls[c].end(), [](const ModexpItem& x, const ModexpItem& y) { return x.exp_len > y.exp_len; });
    items.insert(items.end(), cls[c].begin(), cls[c].end());
    first[c + 1] = (uint32_t)items.size();
  }
  cudaStream_t st = ctx->stream;
  uint8_t *din, *dout;
  ModexpItem* ditems;
  B2_TRY(carve(ctx, ctx->ws_pairing, [&](Carve& c) {
    din = c.take<uint8_t>(in_total);
    ditems = c.take<ModexpItem>(items.size());
    dout = c.take<uint8_t>(out_total);
  }));
  if (in_total) B2_CUDA(ctx, cudaMemcpyAsync(din, data, in_total, cudaMemcpyHostToDevice, st));
  if (!items.empty()) B2_CUDA(ctx, cudaMemcpyAsync(ditems, items.data(), items.size() * sizeof(ModexpItem), cudaMemcpyHostToDevice, st));
  if (out_total) B2_CUDA(ctx, cudaMemsetAsync(dout, 0, out_total, st));
  for (int c = 0; c < kClasses; ++c) {
    const uint32_t n = first[c + 1] - first[c];
    if (!n) continue;
    const ModexpItem* di = ditems + first[c];
    switch (c) {
      case 0: B2_TRY(launch_class<8>(ctx, st, din, di, n, dout)); break;
      case 1: B2_TRY(launch_class<32>(ctx, st, din, di, n, dout)); break;
      case 2: B2_TRY(launch_class<64>(ctx, st, din, di, n, dout)); break;
      case 3: B2_TRY(launch_class<128>(ctx, st, din, di, n, dout)); break;
      default: B2_TRY(launch_class<256>(ctx, st, din, di, n, dout)); break;
    }
  }
  if (out_total) B2_CUDA(ctx, cudaMemcpyAsync(out, dout, out_total, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

}  // extern "C"
