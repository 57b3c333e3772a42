// Exploration probe (not the product): a carry-flag-free Montgomery product on 9 x 29-bit limbs against the
// shipped 8 x 32-bit carry-chain product (csrc/field.cuh), and the raw issue rates behind the difference.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -I ethrex_b200/csrc -o tools/build/mul29_probe tools/mul29_probe.cu
//   tools/build/mul29_probe cpu   -> prints test vectors (hex) for a big-integer check, no GPU needed
//   tools/build/mul29_probe       -> throughput on the GPU
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <cuda_runtime.h>
#include "field.cuh"

#define HD __host__ __device__ __forceinline__
static constexpr uint32_t MASK29 = (1u << 29) - 1;
static constexpr uint32_t PINV29 = 0x4866389u;  // -p^-1 mod 2^29
HD constexpr uint32_t P29(int i) {
  constexpr uint32_t p[9] = {0x187cfd47u, 0x10460b6u, 0x1c72a34fu, 0x2d522d0u, 0x1585d978u, 0x2db40c0u, 0xa6e141u, 0xe5c2634u, 0x30644eu};
  return p[i];
}
struct F29 { uint32_t v[9]; };

// a * b / 2^261 mod p, inputs and output canonical (< p), limbs < 2^29.  Only 64-bit multiply-adds: no carry flags.
HD F29 mul29(const F29& a, const F29& b) {
  uint64_t t[9];
#pragma unroll
  for (int j = 0; j < 9; ++j) t[j] = 0;
#pragma unroll
  for (int i = 0; i < 9; ++i) {
#pragma unroll
    for (int j = 0; j < 9; ++j) t[j] += (uint64_t)a.v[j] * b.v[i];
    uint32_t m = ((uint32_t)t[0] * PINV29) & MASK29;
#pragma unroll
    for (int j = 0; j < 9; ++j) t[j] += (uint64_t)m * P29(j);
    uint64_t c = t[0] >> 29;
#pragma unroll
    for (int j = 0; j < 8; ++j) t[j] = t[j + 1];
    t[0] += c;
    t[8] = 0;
  }
  // carry-normalise to 29-bit limbs (value < 2p)
  F29 r;
  uint64_t c = 0;
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    uint64_t s = t[j] + c;
    r.v[j] = (uint32_t)s & MASK29;
    c = s >> 29;
  }
  // conditional subtraction of p, borrow carried in the sign of a 32-bit difference
  uint32_t d[9];
  int32_t br = 0;
#pragma unroll
  for (int j = 0; j < 9; ++j) {
    int32_t x = (int32_t)r.v[j] - (int32_t)P29(j) + br;
    d[j] = (uint32_t)x & MASK29;
    br = x >> 29;  // 0 or -1
  }
#pragma unroll
  for (int j = 0; j < 9; ++j) r.v[j] = br ? r.v[j] : d[j];
  return r;
}

// ---------------------------------------------------------------------------------------------------------------
static uint64_t sm64(uint64_t& s) { s += 0x9e3779b97f4a7c15ull; uint64_t z = s; z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull; z = (z ^ (z >> 27)) * 0x94d049bb133111ebull; return z ^ (z >> 31); }

__global__ void __launch_bounds__(256) k_mul29(const uint32_t* in, uint32_t* out, int rep) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  F29 a, b, c, d;
  for (int k = 0; k < 9; ++k) { a.v[k] = in[i * 36 + k]; b.v[k] = in[i * 36 + 9 + k]; c.v[k] = in[i * 36 + 18 + k]; d.v[k] = in[i * 36 + 27 + k]; }
  for (int r = 0; r < rep; ++r) { a = mul29(a, b); c = mul29(c, d); b = mul29(b, a); d = mul29(d, c); }
  for (int k = 0; k < 9; ++k) out[i * 9 + k] = a.v[k] ^ b.v[k] ^ c.v[k] ^ d.v[k];
}
__global__ void __launch_bounds__(256) k_mul32(const uint32_t* in, uint32_t* out, int rep) {
  using b200zk::Fq;
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  Fq a, b, c, d;
  for (int k = 0; k < 8; ++k) { a.v[k] = in[i * 36 + k]; b.v[k] = in[i * 36 + 9 + k]; c.v[k] = in[i * 36 + 18 + k]; d.v[k] = in[i * 36 + 27 + k]; }
  a.v[7] &= 0x0fffffff; b.v[7] &= 0x0fffffff; c.v[7] &= 0x0fffffff; d.v[7] &= 0x0fffffff;
  for (int r = 0; r < rep; ++r) { a = Fq::mul(a, b); c = Fq::mul(c, d); b = Fq::mul(b, a); d = Fq::mul(d, c); }
  for (int k = 0; k < 8; ++k) out[i * 9 + k] = a.v[k] ^ b.v[k] ^ c.v[k] ^ d.v[k];
}
// raw rates: 64-bit multiply-add without flags vs the lo.cc / hi.cc carry chain of field.cuh
__global__ void __launch_bounds__(256) k_wide(uint32_t* out, int iters, uint32_t a0) {
  uint64_t acc[8];
  uint32_t a = a0 + threadIdx.x, b = a0 * 3 + blockIdx.x;
  for (int i = 0; i < 8; ++i) acc[i] = i + 977u * threadIdx.x;
  for (int it = 0; it < iters; ++it) {
    a ^= (uint32_t)acc[0]; b += (uint32_t)(acc[0] >> 32);  // loop-variant operands: nothing to hoist
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int i = 0; i < 8; ++i) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i]) : "r"((uint32_t)acc[(i + 1) & 7]), "r"(b));
  }
  uint64_t r = 0;
  for (int i = 0; i < 8; ++i) r ^= acc[i];
  if (r == 0x1234567ull) out[0] = (uint32_t)r;
}
// operand-pattern variants of the flag-free multiply-add: does the rate survive distinct source registers?
template <int MODE>
__global__ void __launch_bounds__(256) k_wide_var(uint32_t* out, int iters, uint32_t a0) {
  uint64_t acc[8];
  uint32_t a[8], b[8];
  for (int i = 0; i < 8; ++i) { acc[i] = i + 977u * threadIdx.x; a[i] = a0 * (i + 3) + threadIdx.x; b[i] = a0 * (i + 11) + blockIdx.x; }
  for (int it = 0; it < iters; ++it) {
    for (int i = 0; i < 8; ++i) { a[i] ^= (uint32_t)acc[(i + 1) & 7]; b[i] += (uint32_t)(acc[(i + 3) & 7] >> 32); }
#pragma unroll
    for (int u = 0; u < 4; ++u)
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (MODE == 0) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i]) : "r"((uint32_t)acc[(i + 1) & 7]), "r"(b[0]));        // a = neighbour chain, b shared
        if (MODE == 1) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i]) : "r"((uint32_t)acc[(i + 1) & 7]), "r"(b[i]));        // a = neighbour chain, b[i] distinct
        if (MODE == 2) asm volatile("mad.wide.u32 %0, %1, 0x187cfd47, %0;" : "+l"(acc[i]) : "r"((uint32_t)acc[(i + 1) & 7]));           // immediate multiplier
        if (MODE == 3) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i]) : "r"((uint32_t)(acc[(i + 1) & 7] >> 32)), "r"(b[(i * 3 + u) & 7]));  // a = high word of the neighbour
      }
  }
  uint64_t r = 0;
  for (int i = 0; i < 8; ++i) r ^= acc[i];
  if (r == 0x1234567ull) out[0] = (uint32_t)r;
}
__global__ void __launch_bounds__(256) k_chain(uint32_t* out, int iters, uint32_t a0) {
  uint32_t x[8], top = 0;
  uint32_t a = a0 + threadIdx.x, b = a0 * 3 + blockIdx.x;
  for (int i = 0; i < 8; ++i) x[i] = i;
  for (int it = 0; it < iters; ++it)
#pragma unroll
    for (int u = 0; u < 8; ++u) b200zk::detail::mad_even(x, top, a, a ^ 5, a ^ 9, a ^ 17, b);  // 4 wide products in one chain
  uint32_t r = top;
  for (int i = 0; i < 8; ++i) r ^= x[i];
  if (r == 0x1234567u) out[0] = r;
}

template <class K, class... A> static float time_kernel(K k, dim3 g, dim3 b, A... args) {
  k<<<g, b>>>(args...);
  cudaDeviceSynchronize();
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  k<<<g, b>>>(args...);
  cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  return ms;
}

int main(int argc, char** argv) {
  if (argc > 1 && !strcmp(argv[1], "cpu")) {
    uint64_t s = 0xB2000029;
    for (int t = 0; t < 200; ++t) {
      F29 a, b;
      for (int k = 0; k < 9; ++k) { a.v[k] = (uint32_t)sm64(s) & MASK29; b.v[k] = (uint32_t)sm64(s) & MASK29; }
      a.v[8] &= 0x1fffff; b.v[8] &= 0x1fffff;  // < 2^253 < p
      if (t == 0) { for (int k = 0; k < 9; ++k) { a.v[k] = P29(k); b.v[k] = P29(k); } a.v[0] -= 1; b.v[0] -= 1; }  // (p-1)^2
      if (t == 1) { for (int k = 0; k < 9; ++k) a.v[k] = 0; }
      F29 r = mul29(a, b);
      for (int k = 0; k < 9; ++k) printf("%x ", a.v[k]);
      printf("| ");
      for (int k = 0; k < 9; ++k) printf("%x ", b.v[k]);
      printf("| ");
      for (int k = 0; k < 9; ++k) printf("%x ", r.v[k]);
      printf("\n");
    }
    return 0;
  }
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
  const double ghz = khz * 1e-6;
  const int sms = p.multiProcessorCount;
  const size_t n = (size_t)sms * 256 * 16;
  uint32_t *in, *out;
  cudaMalloc(&in, n * 36 * 4); cudaMalloc(&out, n * 9 * 4);
  uint32_t* h = (uint32_t*)malloc(n * 36 * 4);
  uint64_t s = 1;
  for (size_t i = 0; i < n * 36; ++i) h[i] = (uint32_t)sm64(s) & 0x0fffffff;
  cudaMemcpy(in, h, n * 36 * 4, cudaMemcpyHostToDevice);
  const int rep = 256;
  float m29 = time_kernel(k_mul29, dim3(n / 256), dim3(256), in, out, rep);
  float m32 = time_kernel(k_mul32, dim3(n / 256), dim3(256), in, out, rep);
  double prods = (double)n * rep * 4;
  printf("{\"probe\": \"mul29 (9x29, no carry flags)\", \"ms\": %.3f, \"Gmul_per_s\": %.1f, \"clk_per_lane_product\": %.2f}\n", m29, prods / m29 * 1e-6, m29 * 1e-3 * ghz * 1e9 * sms / prods);
  printf("{\"probe\": \"mul32 (field.cuh carry chains)\", \"ms\": %.3f, \"Gmul_per_s\": %.1f, \"clk_per_lane_product\": %.2f}\n", m32, prods / m32 * 1e-6, m32 * 1e-3 * ghz * 1e9 * sms / prods);
  const int iters = 2048;
  float mw = time_kernel(k_wide, dim3(sms * 8), dim3(256), out, iters, 3u);
  float mc = time_kernel(k_chain, dim3(sms * 8), dim3(256), out, iters, 3u);
  double thr = (double)sms * 8 * 256;
  printf("{\"probe\": \"mad.wide.u32 (64-bit accumulate, no flags)\", \"wide_per_clk_sm\": %.1f}\n", thr * iters * 32 / (mw * 1e-3 * ghz * 1e9 * sms));
  printf("{\"probe\": \"mad.lo.cc/madc.hi.cc chain (IMAD.WIDE.X)\", \"wide_per_clk_sm\": %.1f}\n", thr * iters * 32 / (mc * 1e-3 * ghz * 1e9 * sms));
  const char* names[4] = {"mad.wide: a = neighbour chain, b shared", "mad.wide: a = neighbour chain, b[i] distinct", "mad.wide: a = neighbour chain, immediate b", "mad.wide: a = neighbour high word, b rotating"};
  float v0 = time_kernel(k_wide_var<0>, dim3(sms * 8), dim3(256), out, iters, 3u);
  float v1 = time_kernel(k_wide_var<1>, dim3(sms * 8), dim3(256), out, iters, 3u);
  float v2 = time_kernel(k_wide_var<2>, dim3(sms * 8), dim3(256), out, iters, 3u);
  float v3 = time_kernel(k_wide_var<3>, dim3(sms * 8), dim3(256), out, iters, 3u);
  float vs[4] = {v0, v1, v2, v3};
  for (int i = 0; i < 4; ++i) printf("{\"probe\": \"%s\", \"wide_per_clk_sm\": %.1f}\n", names[i], thr * iters * 32 / (vs[i] * 1e-3 * ghz * 1e9 * sms));
  return 0;
}
