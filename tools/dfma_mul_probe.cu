// Exploration probe (not the product): a 254-bit Montgomery product built on the FP64 pipe (DFMA) against the
// shipped 8 x 32-bit IMAD.WIDE carry-chain product of csrc/field.cuh.  VERDICT r1 "next" item 3.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -I ethrex_b200/csrc -Xcompiler -frounding-math \
//        -o tools/build/dfma_mul_probe tools/dfma_mul_probe.cu
//   tools/build/dfma_mul_probe cpu [count]   host run of the SAME code (fma() under FE_TOWARDZERO): prints
//                                             "a b r" hex triples for the big-integer check in tools/dfma_check.py
//   tools/build/dfma_mul_probe               GPU: bit-exactness of the device path against the host path on the
//                                             same vectors, then throughput of every variant (JSON lines)
//
// Representation: 5 limbs of 52 bits (uint64), Montgomery radix R = 2^260, values < 2p (mul returns < p when CANON).
// Emmart/Zheng/Weems split of a 52 x 52-bit product with two FMAs and one exact addition, all on the FP64 pipe:
//     hi = fma.rz(a, b, 2^104)                -> mantissa(hi) = floor(a*b / 2^52)
//     lo = fma.rz(a, b, (2^104 + 2^52) - hi)  -> mantissa(lo) = a*b mod 2^52            (exact: the sum is in [2^52, 2^53))
// The raw IEEE bit patterns are accumulated as 64-bit integers; their exponent fields (0x467 / 0x433) are constants
// whose column totals are folded into the accumulators' initial values, and they never touch the low 52 bits the
// Montgomery quotient digit is read from.
#include <cfenv>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <cuda_runtime.h>
#include "field.cuh"

#define HD __host__ __device__ __forceinline__

static constexpr uint64_t M52 = (1ull << 52) - 1;
HD constexpr uint64_t P52(int i) {
  constexpr uint64_t p[5] = {0x8c16d87cfd47ull, 0x916871ca8d3c2ull, 0x181585d97816aull, 0xa029b85045b68ull, 0x30644e72e131ull};
  return p[i];
}
static constexpr uint64_t PINV52 = 0x20782e4866389ull;  // -p^-1 mod 2^52
// -(n_lo(c) * 0x433<<52 + n_hi(c) * 0x467<<52) mod 2^64: column c receives n_lo = 2*cnt(c) low halves and
// n_hi = 2*cnt(c-1) high halves over the whole product (a*b and m*p), cnt(c) = #{(i,j): i+j = c}
HD constexpr uint64_t BIAS0(int c) {
  constexpr uint64_t b[10] = {0x79a0000000000000ull, 0x6660000000000000ull, 0x5320000000000000ull, 0x3fe0000000000000ull, 0x2ca0000000000000ull,
                              0x2620000000000000ull, 0x3960000000000000ull, 0x4ca0000000000000ull, 0x5fe0000000000000ull, 0x7320000000000000ull};
  return b[c];
}

struct F52 { uint64_t v[5]; };

HD double fma_rz(double a, double b, double c) {
#ifdef __CUDA_ARCH__
  return __fma_rz(a, b, c);
#else
  return std::fma(a, b, c);  // the host harness runs under fesetround(FE_TOWARDZERO)
#endif
}
HD uint64_t d2u(double x) {
#ifdef __CUDA_ARCH__
  return (uint64_t)__double_as_longlong(x);
#else
  uint64_t u; memcpy(&u, &x, 8); return u;
#endif
}
HD double u2d_bits(uint64_t u) {
#ifdef __CUDA_ARCH__
  return __longlong_as_double((long long)u);
#else
  double x; memcpy(&x, &u, 8); return x;
#endif
}
// integer < 2^52 -> double, without the conversion unit: splice it under the exponent of 2^52 and subtract 2^52 (exact)
HD double u2d(uint64_t x) { return u2d_bits(x | 0x4330000000000000ull) - 4503599627370496.0; }

// acc[c] += low half, acc[c + 1] += high half of a * b  (a, b < 2^52 as doubles)
HD void split_acc(uint64_t* acc, int c, double a, double b) {
  const double C1 = 20282409603651670423947251286016.0;                      // 2^104
  const double C2 = 20282409603651670423947251286016.0 + 4503599627370496.0;  // 2^104 + 2^52
  double hi = fma_rz(a, b, C1);
  double lo = fma_rz(a, b, C2 - hi);
  acc[c] += d2u(lo);
  acc[c + 1] += d2u(hi);
}

// a * b / 2^260 mod p.  Inputs < 2^3 p (limbs < 2^52), output < 2p, or < p with CANON.
template <bool CANON>
HD F52 mul52(const F52& a, const F52& b) {
  double ad[5], bd[5];
#pragma unroll
  for (int i = 0; i < 5; ++i) { ad[i] = u2d(a.v[i]); bd[i] = u2d(b.v[i]); }
  uint64_t acc[10];
#pragma unroll
  for (int c = 0; c < 10; ++c) acc[c] = BIAS0(c);
#pragma unroll
  for (int i = 0; i < 5; ++i) {
#pragma unroll
    for (int j = 0; j < 5; ++j) split_acc(acc, i + j, ad[j], bd[i]);
    const uint64_t m = ((acc[i] & M52) * PINV52) & M52;
    const double md = u2d(m);
#pragma unroll
    for (int j = 0; j < 5; ++j) split_acc(acc, i + j, md, (double)P52(j));
    acc[i + 1] += acc[i] >> 52;  // column i is complete and == 0 mod 2^52: pass its carry on
  }
  F52 r;
  uint64_t t = acc[5];
#pragma unroll
  for (int k = 0; k < 4; ++k) { r.v[k] = t & M52; t = acc[6 + k] + (t >> 52); }
  r.v[4] = t;
  if (CANON) {
    uint64_t d[5];
    int64_t br = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      int64_t x = (int64_t)r.v[k] - (int64_t)P52(k) + br;
      d[k] = (uint64_t)x & M52;
      br = x >> 63;
    }
#pragma unroll
    for (int k = 0; k < 5; ++k) r.v[k] = br ? r.v[k] : d[k];
  }
  return r;
}

// a^2 / 2^260 mod p: the 10 off-diagonal limb products are issued once against the doubled operand (2 a_j < 2^53 is
// still exact, but the split needs both factors < 2^52, so the doubling is applied to the ACCUMULATED halves instead:
// off-diagonal halves are summed in their own accumulators and added twice).
template <bool CANON>
HD F52 sqr52(const F52& a) {
  double ad[5];
#pragma unroll
  for (int i = 0; i < 5; ++i) ad[i] = u2d(a.v[i]);
  // off-diagonal part X = sum_{i<j} a_i a_j 2^(52(i+j)) as raw-biased columns, then acc = 2X + diag + reduction
  uint64_t off[10];
#pragma unroll
  for (int c = 0; c < 10; ++c) off[c] = 0;
#pragma unroll
  for (int i = 0; i < 5; ++i)
#pragma unroll
    for (int j = i + 1; j < 5; ++j) split_acc(off, i + j, ad[i], ad[j]);
  uint64_t acc[10];
#pragma unroll
  for (int c = 0; c < 10; ++c) acc[c] = BIAS0(c) + 2 * off[c];
#pragma unroll
  for (int i = 0; i < 5; ++i) split_acc(acc, 2 * i, ad[i], ad[i]);
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    const uint64_t m = ((acc[i] & M52) * PINV52) & M52;
    const double md = u2d(m);
#pragma unroll
    for (int j = 0; j < 5; ++j) split_acc(acc, i + j, md, (double)P52(j));
    acc[i + 1] += acc[i] >> 52;
  }
  F52 r;
  uint64_t t = acc[5];
#pragma unroll
  for (int k = 0; k < 4; ++k) { r.v[k] = t & M52; t = acc[6 + k] + (t >> 52); }
  r.v[4] = t;
  if (CANON) {
    uint64_t d[5];
    int64_t br = 0;
#pragma unroll
    for (int k = 0; k < 5; ++k) {
      int64_t x = (int64_t)r.v[k] - (int64_t)P52(k) + br;
      d[k] = (uint64_t)x & M52;
      br = x >> 63;
    }
#pragma unroll
    for (int k = 0; k < 5; ++k) r.v[k] = br ? r.v[k] : d[k];
  }
  return r;
}

// ---------------------------------------------------------------------------------------------------------------
static uint64_t sm64(uint64_t& s) { s += 0x9e3779b97f4a7c15ull; uint64_t z = s; z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull; z = (z ^ (z >> 27)) * 0x94d049bb133111ebull; return z ^ (z >> 31); }

static bool geq_p(const F52& a) {
  for (int k = 4; k >= 0; --k) { if (a.v[k] != P52(k)) return a.v[k] > P52(k); }
  return true;
}
static F52 rand_below_p(uint64_t& s) {
  F52 a;
  do {
    for (int k = 0; k < 5; ++k) a.v[k] = sm64(s) & M52;
    a.v[4] &= (1ull << 46) - 1;  // 254 bits
  } while (geq_p(a));
  return a;
}
static F52 from_small(uint64_t x) { F52 a = {{x & M52, x >> 52, 0, 0, 0}}; return a; }
static F52 p_minus(uint64_t k) {  // p - k, k small
  F52 a; for (int i = 0; i < 5; ++i) a.v[i] = P52(i);
  a.v[0] -= k; return a;
}
static void edge_set(std::vector<F52>& e) {
  e.push_back(from_small(0)); e.push_back(from_small(1)); e.push_back(from_small(2)); e.push_back(from_small(M52));
  e.push_back(p_minus(1)); e.push_back(p_minus(2));
  F52 ones; for (int i = 0; i < 5; ++i) ones.v[i] = M52; ones.v[4] = P52(4) - 1; e.push_back(ones);  // all-ones low limbs, < p
  F52 hi = from_small(0); hi.v[4] = P52(4); e.push_back(hi);  // only the top limb
  F52 alt; for (int i = 0; i < 5; ++i) alt.v[i] = (i & 1) ? M52 : 0; alt.v[4] = 0; e.push_back(alt);
  F52 alt2; for (int i = 0; i < 5; ++i) alt2.v[i] = (i & 1) ? 0 : M52; alt2.v[4] = 1; e.push_back(alt2);
  F52 pw; for (int i = 0; i < 5; ++i) pw.v[i] = 1ull << 51; pw.v[4] = 1ull << 44; e.push_back(pw);
}
static void make_vectors(size_t count, std::vector<F52>& A, std::vector<F52>& B) {
  std::vector<F52> e; edge_set(e);
  for (auto& x : e) for (auto& y : e) { A.push_back(x); B.push_back(y); }
  uint64_t s = 0xB2005200ull;
  while (A.size() < count) { A.push_back(rand_below_p(s)); B.push_back(rand_below_p(s)); }
}
static void print52(const F52& a) {  // 260-bit value as hex
  // limbs of 52 bits = 13 hex digits each
  printf("%013llx%013llx%013llx%013llx%013llx", (unsigned long long)a.v[4], (unsigned long long)a.v[3], (unsigned long long)a.v[2], (unsigned long long)a.v[1], (unsigned long long)a.v[0]);
}

__global__ void k_check(const F52* A, const F52* B, F52* R, F52* S, size_t n) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  R[i] = mul52<true>(A[i], B[i]);
  S[i] = sqr52<true>(A[i]);
}

template <int MODE>  // 0: mul52 canonical, 1: mul52 lazy (< 2p), 2: sqr52 canonical, 3: sqr52 lazy
__global__ void __launch_bounds__(256) k_mul52(const uint64_t* in, uint64_t* out, int rep) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  F52 a, b, c, d;
  for (int k = 0; k < 5; ++k) { a.v[k] = in[i * 20 + k] & M52; b.v[k] = in[i * 20 + 5 + k] & M52; c.v[k] = in[i * 20 + 10 + k] & M52; d.v[k] = in[i * 20 + 15 + k] & M52; }
  a.v[4] &= (1ull << 45) - 1; b.v[4] &= (1ull << 45) - 1; c.v[4] &= (1ull << 45) - 1; d.v[4] &= (1ull << 45) - 1;
  for (int r = 0; r < rep; ++r) {
    if (MODE == 0) { a = mul52<true>(a, b); c = mul52<true>(c, d); b = mul52<true>(b, a); d = mul52<true>(d, c); }
    if (MODE == 1) { a = mul52<false>(a, b); c = mul52<false>(c, d); b = mul52<false>(b, a); d = mul52<false>(d, c); }
    if (MODE == 2) { a = sqr52<true>(a); c = sqr52<true>(c); b = sqr52<true>(b); d = sqr52<true>(d); }
    if (MODE == 3) { a = sqr52<false>(a); c = sqr52<false>(c); b = sqr52<false>(b); d = sqr52<false>(d); }
  }
  for (int k = 0; k < 5; ++k) out[i * 5 + k] = a.v[k] ^ b.v[k] ^ c.v[k] ^ d.v[k];
}
// the lazy product again under a 64-register cap (4 CTAs of 256 threads per SM instead of 3): is it occupancy?
__global__ void __launch_bounds__(256, 4) k_mul52_r64(const uint64_t* in, uint64_t* out, int rep) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  F52 a, b, c, d;
  for (int k = 0; k < 5; ++k) { a.v[k] = in[i * 20 + k] & M52; b.v[k] = in[i * 20 + 5 + k] & M52; c.v[k] = in[i * 20 + 10 + k] & M52; d.v[k] = in[i * 20 + 15 + k] & M52; }
  a.v[4] &= (1ull << 45) - 1; b.v[4] &= (1ull << 45) - 1; c.v[4] &= (1ull << 45) - 1; d.v[4] &= (1ull << 45) - 1;
  for (int r = 0; r < rep; ++r) { a = mul52<false>(a, b); c = mul52<false>(c, d); b = mul52<false>(b, a); d = mul52<false>(d, c); }
  for (int k = 0; k < 5; ++k) out[i * 5 + k] = a.v[k] ^ b.v[k] ^ c.v[k] ^ d.v[k];
}
// two independent products per thread instead of four interleaved chains: fewer live registers, less ILP
__global__ void __launch_bounds__(256) k_mul52_ilp2(const uint64_t* in, uint64_t* out, int rep) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  F52 a, b;
  for (int k = 0; k < 5; ++k) { a.v[k] = in[i * 20 + k] & M52; b.v[k] = in[i * 20 + 5 + k] & M52; }
  a.v[4] &= (1ull << 45) - 1; b.v[4] &= (1ull << 45) - 1;
  for (int r = 0; r < 2 * rep; ++r) { a = mul52<false>(a, b); b = mul52<false>(b, a); }
  for (int k = 0; k < 5; ++k) out[i * 5 + k] = a.v[k] ^ b.v[k];
}

template <int MODE>  // 0: Fq::mul, 1: Fq::sqr  (the shipped product, same harness)
__global__ void __launch_bounds__(256) k_mul32(const uint64_t* in64, uint64_t* out64, int rep) {
  using b200zk::Fq;
  const uint32_t* in = reinterpret_cast<const uint32_t*>(in64);
  uint32_t* out = reinterpret_cast<uint32_t*>(out64);
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  Fq a, b, c, d;
  for (int k = 0; k < 8; ++k) { a.v[k] = in[i * 40 + k]; b.v[k] = in[i * 40 + 8 + k]; c.v[k] = in[i * 40 + 16 + k]; d.v[k] = in[i * 40 + 24 + k]; }
  a.v[7] &= 0x0fffffff; b.v[7] &= 0x0fffffff; c.v[7] &= 0x0fffffff; d.v[7] &= 0x0fffffff;
  for (int r = 0; r < rep; ++r) {
    if (MODE == 0) { a = Fq::mul(a, b); c = Fq::mul(c, d); b = Fq::mul(b, a); d = Fq::mul(d, c); }
    else { a = Fq::sqr(a); c = Fq::sqr(c); b = Fq::sqr(b); d = Fq::sqr(d); }
  }
  for (int k = 0; k < 8; ++k) out[i * 10 + k] = a.v[k] ^ b.v[k] ^ c.v[k] ^ d.v[k];
}

int main(int argc, char** argv) {
  fesetround(FE_TOWARDZERO);
  if (argc > 1 && !strcmp(argv[1], "cpu")) {
    size_t count = argc > 2 ? strtoull(argv[2], nullptr, 10) : 10000;
    std::vector<F52> A, B; make_vectors(count, A, B);
    for (size_t i = 0; i < A.size(); ++i) {
      F52 r = mul52<true>(A[i], B[i]), s = sqr52<true>(A[i]);
      print52(A[i]); printf(" "); print52(B[i]); printf(" "); print52(r); printf(" "); print52(s); printf("\n");
    }
    return 0;
  }
  int dev = 0; cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess) { fprintf(stderr, "no CUDA device\n"); return 2; }
  // ---- bit-exactness: device against host on the same vectors (the host path is checked against big integers by tools/dfma_check.py)
  {
    std::vector<F52> A, B; make_vectors(20000, A, B);
    const size_t n = A.size();
    F52 *dA, *dB, *dR, *dS;
    cudaMalloc(&dA, n * sizeof(F52)); cudaMalloc(&dB, n * sizeof(F52)); cudaMalloc(&dR, n * sizeof(F52)); cudaMalloc(&dS, n * sizeof(F52));
    cudaMemcpy(dA, A.data(), n * sizeof(F52), cudaMemcpyHostToDevice); cudaMemcpy(dB, B.data(), n * sizeof(F52), cudaMemcpyHostToDevice);
    k_check<<<(unsigned)((n + 127) / 128), 128>>>(dA, dB, dR, dS, n);
    std::vector<F52> R(n), S(n);
    cudaMemcpy(R.data(), dR, n * sizeof(F52), cudaMemcpyDeviceToHost); cudaMemcpy(S.data(), dS, n * sizeof(F52), cudaMemcpyDeviceToHost);
    size_t bad = 0;
    for (size_t i = 0; i < n; ++i) {
      F52 r = mul52<true>(A[i], B[i]), s = sqr52<true>(A[i]);
      if (memcmp(&r, &R[i], sizeof r) || memcmp(&s, &S[i], sizeof s)) ++bad;
    }
    printf("{\"probe\": \"dfma_bit_exact\", \"vectors\": %zu, \"mismatches\": %zu, \"cuda\": \"%s\"}\n", n, bad, cudaGetErrorString(cudaGetLastError()));
    cudaFree(dA); cudaFree(dB); cudaFree(dR); cudaFree(dS);
    if (bad) return 1;
  }
  // ---- throughput
  const int ctas = prop.multiProcessorCount * 8, threads = 256, rep = 256;
  const size_t n = (size_t)ctas * threads;
  std::vector<uint64_t> h(n * 20);
  uint64_t s = 0x5eed;
  for (auto& x : h) x = sm64(s);
  uint64_t *din, *dout;
  cudaMalloc(&din, h.size() * 8); cudaMalloc(&dout, n * 5 * 8);
  cudaMemcpy(din, h.data(), h.size() * 8, cudaMemcpyHostToDevice);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  int clk_khz = 0; cudaDeviceGetAttribute(&clk_khz, cudaDevAttrClockRate, dev);
  auto run = [&](const char* name, auto kernel) {
    kernel<<<ctas, threads>>>(din, dout, 8);  // warm-up
    cudaDeviceSynchronize();
    float best = 1e30f;
    for (int t = 0; t < 5; ++t) {
      cudaEventRecord(e0);
      kernel<<<ctas, threads>>>(din, dout, rep);
      cudaEventRecord(e1); cudaEventSynchronize(e1);
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      if (ms < best) best = ms;
    }
    double products = (double)n * rep * 4;
    double gps = products / (best * 1e-3) / 1e9;
    double sm_clk = (double)prop.multiProcessorCount * (clk_khz * 1e3) / (gps * 1e9);  // SM-clocks per lane-product at the nominal max clock
    printf("{\"probe\": \"%s\", \"ms\": %.4f, \"G_products_per_s\": %.2f, \"sm_clocks_per_product_at_max_clock\": %.3f, \"err\": \"%s\"}\n", name, best, gps, sm_clk,
           cudaGetErrorString(cudaGetLastError()));
  };
  run("mul32_field_cuh (IMAD.WIDE carry chains, R=2^256)", k_mul32<0>);
  run("sqr32_field_cuh", k_mul32<1>);
  run("mul52_dfma canonical (<p)", k_mul52<0>);
  run("mul52_dfma lazy (<2p, no final subtraction)", k_mul52<1>);
  run("mul52_dfma lazy, 64-register cap (4 CTAs/SM)", k_mul52_r64);
  run("mul52_dfma lazy, 2 chains per thread", k_mul52_ilp2);
  run("sqr52_dfma canonical", k_mul52<2>);
  run("sqr52_dfma lazy", k_mul52<3>);
  return 0;
}
