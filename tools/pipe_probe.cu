// Pipe probe (exploration, not the product): do IMAD.WIDE (fmaheavy pipe) and DFMA (fp64 pipe) issue concurrently
// on sm_90a, and at what rates?  Decides whether a double-precision limb product can run beside the integer one.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/build/pipe_probe tools/pipe_probe.cu && tools/build/pipe_probe
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

template <int NI, int ND>
__global__ void __launch_bounds__(256) probe(uint64_t* out, int iters, uint32_t a0, double d0) {
  uint64_t acc[NI > 0 ? NI : 1];
  double dac[ND > 0 ? ND : 1];
  uint32_t a = a0 + threadIdx.x, b = a0 * 3 + blockIdx.x;
  double da = d0 + threadIdx.x, db = d0 * 0.5;
#pragma unroll
  for (int i = 0; i < NI; ++i) acc[i] = i + 977u * threadIdx.x;
#pragma unroll
  for (int i = 0; i < ND; ++i) dac[i] = i + 0.37 * threadIdx.x;
  for (int it = 0; it < iters; ++it) {
    // the operands must change every iteration: with loop-invariant a, b ptxas hoists the product out of the loop
    // and the "multiply-add" degenerates into a 64-bit add (the first version of this probe measured exactly that)
    if (NI) { a ^= (uint32_t)acc[0]; b += (uint32_t)(acc[0] >> 32); }
    if (ND) { da += dac[0] * 1e-300; }
#pragma unroll
    for (int u = 0; u < 8; ++u) {
#pragma unroll
      for (int i = 0; i < (NI > ND ? NI : ND); ++i) {
        // the multiplicand is the neighbour chain's running value: no two products are alike, nothing can be CSE'd
        if (i < NI) asm volatile("mad.wide.u32 %0, %1, %2, %0;" : "+l"(acc[i]) : "r"((uint32_t)acc[(i + 1) % (NI > 0 ? NI : 1)]), "r"(b));
        if (i < ND) asm volatile("fma.rn.f64 %0, %1, %2, %0;" : "+d"(dac[i]) : "d"(dac[(i + 1) % (ND > 0 ? ND : 1)]), "d"(db));
      }
    }
  }
  uint64_t r = 0;
#pragma unroll
  for (int i = 0; i < NI; ++i) r ^= acc[i];
#pragma unroll
  for (int i = 0; i < ND; ++i) r ^= (uint64_t)__double_as_longlong(dac[i]);
  if (r == 0x1234567ull) out[0] = r;
}

template <int NI, int ND>
static void run(const char* name, int sms, double ghz) {
  uint64_t* d;
  cudaMalloc(&d, 8);
  const int iters = 4096, grid = sms * 8;
  probe<NI, ND><<<grid, 256>>>(d, 16, 3, 1.5);
  cudaDeviceSynchronize();
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  cudaEventRecord(e0);
  probe<NI, ND><<<grid, 256>>>(d, iters, 3, 1.5);
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  double threads = (double)grid * 256, per = (double)iters * 8;
  double imad = threads * per * NI, dfma = threads * per * ND;
  double clk = ms * 1e-3 * ghz * 1e9 * sms;  // SM-cycles
  printf("{\"probe\": \"%s\", \"ms\": %.3f, \"imad_wide_per_clk_sm\": %.1f, \"dfma_per_clk_sm\": %.1f, \"imad_T/s\": %.2f, \"dfma_T/s\": %.2f}\n",
         name, ms, imad / clk, dfma / clk, imad / ms * 1e-9, dfma / ms * 1e-9);
  cudaFree(d);
}

int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  int khz = 0; cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, 0);
  double ghz = khz * 1e-6;
  printf("{\"gpu\": \"%s\", \"sms\": %d, \"clock_ghz_nominal\": %.3f}\n", p.name, p.multiProcessorCount, ghz);
  run<8, 0>("imad_only", p.multiProcessorCount, ghz);
  run<0, 8>("dfma_only", p.multiProcessorCount, ghz);
  run<8, 8>("imad8_dfma8", p.multiProcessorCount, ghz);
  run<4, 8>("imad4_dfma8", p.multiProcessorCount, ghz);
  run<8, 4>("imad8_dfma4", p.multiProcessorCount, ghz);
  run<8, 2>("imad8_dfma2", p.multiProcessorCount, ghz);
  return 0;
}
