// bigmod_conformance.cu -- test-only harness: every primitive of bigmod.cuh at every width modexp.cu instantiates, so
// tests/test_gpu_bigmod_conformance.py can compare each of them with Python integers at the lane edges where carries
// and borrows cross lanes.  Linked into the same test library as field_conformance.cu and built by
// ethrex_b200/csrc/Makefile with the product's own nvcc flags.
//
// One item per group of TPI = N / 8 lanes, launched in blocks of 64 threads as modexp.cu launches its kernel; the groups
// past the last item leave at once, as there.  Item i reads in[i * (1 + 3N) ..]: word 0 is the op id (read per item, so
// the groups of one warp may run different ops), then three operand slots of N little-endian words; a scalar operand
// (cond_sub's hi, truncate_bits' s, neg_inv32's x) is the first word of its slot.  Item i writes out[i * (N + 2) ..]:
// the number result in words 0 .. N-1, the scalar result (carry, borrow, flag, neg_inv32) in word N, as lane 0 has it,
// and in word N + 1 the count of the group's lanes whose scalar differs from lane 0's.  An op leaves the words it does
// not produce untouched.
#include "bigmod.cuh"

using namespace b200zk;
using namespace b200zk::bigmod;

namespace {

enum : int { B_ADD = 0, B_SUB, B_MOD_ADD, B_MOD_DBL, B_COND_SUB, B_MONT_MUL, B_LO_MUL, B_INV_MOD_R, B_TRUNCATE_BITS, B_IS_ZERO,
             B_IS_ONE, B_NEG_INV32, N_BIGMOD_OPS };

constexpr int kThreads = 64;  // modexp.cu's kModexpThreads

template <int N, int TPI>
__global__ void __launch_bounds__(kThreads) bigmod_kernel(const uint32_t* __restrict__ in, uint32_t* __restrict__ out, uint64_t n) {
  static_assert(N == kLimbs * TPI, "eight limbs per lane");
  const Group<TPI> g;
  const uint64_t idx = (uint64_t)blockIdx.x * (kThreads / TPI) + threadIdx.x / TPI;
  if (idx >= n) return;  // the whole group leaves together
  in += idx * (1 + 3 * N);
  out += idx * (N + 2);
  auto num = [&](int k) {
    Num<TPI> a;
#pragma unroll
    for (int j = 0; j < kLimbs; ++j) a.v[j] = in[1 + k * N + g.lane * kLimbs + j];
    return a;
  };
  auto word = [&](int k) { return in[1 + k * N]; };
  auto put = [&](const Num<TPI>& a) {
#pragma unroll
    for (int j = 0; j < kLimbs; ++j) out[g.lane * kLimbs + j] = a.v[j];
  };
  auto scalar = [&](uint32_t w) {
    const uint32_t w0 = g.bcast(w, 0);
    const uint32_t differ = (uint32_t)__popcll(g.ballot(w != w0));
    if (g.lane == 0) {
      out[N] = w0;
      out[N + 1] = differ;
    }
  };
  switch (in[0]) {
    case B_ADD: { Num<TPI> a = num(0); scalar(add(a, num(1), g)); put(a); break; }
    case B_SUB: { Num<TPI> a = num(0); scalar(sub(a, num(1), g)); put(a); break; }
    case B_MOD_ADD: { Num<TPI> a = num(0); mod_add(a, num(1), num(2), g); put(a); break; }
    case B_MOD_DBL: { Num<TPI> a = num(0); mod_dbl(a, num(1), g); put(a); break; }
    case B_COND_SUB: { Num<TPI> t = num(0); cond_sub(t, word(2), num(1), g); put(t); break; }
    case B_MONT_MUL: {  // m' from lane 0, as modexp.cu takes it
      const Num<TPI> m = num(2);
      put(mont_mul(num(0), num(1), m, g.bcast(neg_inv32(m.v[0]), 0), g));
      break;
    }
    case B_LO_MUL: put(lo_mul(num(0), num(1), g)); break;
    case B_INV_MOD_R: put(inv_mod_r(num(0), g)); break;
    case B_TRUNCATE_BITS: { Num<TPI> a = num(0); truncate_bits(a, word(1), g); put(a); break; }
    case B_IS_ZERO: scalar(is_zero(num(0), g) ? 1u : 0u); break;
    case B_IS_ONE: scalar(is_one(num(0), g) ? 1u : 0u); break;
    case B_NEG_INV32: scalar(neg_inv32(word(0))); break;
  }
}

template <int N> void launch(const uint32_t* in, uint32_t* out, uint64_t n) {
  constexpr int per_block = kThreads / (N / kLimbs);
  bigmod_kernel<N, N / kLimbs><<<(uint32_t)((n + per_block - 1) / per_block), kThreads>>>(in, out, n);
}

}  // namespace

// Runs n items of width `limbs` (device pointers, the layout above) on the legacy default stream and waits for it.
// 0 on success, -1 for a width modexp.cu does not instantiate, else the CUDA error code.
extern "C" int b200zk_bigmod_conformance_run(uint32_t limbs, const uint32_t* in, uint32_t* out, uint64_t n) {
  if (limbs != 8 && limbs != 32 && limbs != 64 && limbs != 128 && limbs != 256) return -1;
  if (n == 0) return 0;
  switch (limbs) {
    case 8: launch<8>(in, out, n); break;
    case 32: launch<32>(in, out, n); break;
    case 64: launch<64>(in, out, n); break;
    case 128: launch<128>(in, out, n); break;
    default: launch<256>(in, out, n); break;
  }
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  return (int)e;
}
