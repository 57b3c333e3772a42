// pairing_conformance.cu -- test-only harness: each stage of the two pairings alone, one item per thread, so
// tests/test_gpu_pairing_conformance.py can compare every intermediate value with the Python restatement of
// tests/pairing_stages_ref.py, and the subgroup check with points of every cofactor order.
// Not part of libb200zk.so; ethrex_b200/csrc/Makefile links it into the conformance library with the product's own nvcc
// flags, and it reaches the stages through the same headers the product's kernels are built from (bls_pairing.cuh,
// bn_pairing.cuh, curve.cuh), so the code under test is generated exactly as the library's is.
//
// Layout, as in field_conformance.cu: item i reads in[i * in_words ..] and writes out[i * out_words ..]; every value is
// its raw limbs in the type's own form (Montgomery field elements; an extension element is its coefficients in tower
// order, c0 before c1).  Per op, in words (BLS12-381: Fp 12, Fp2 24, Fp12 288; BN254: Fq 8, Fq2 16, Fq12 192):
//   BLS  FROB, FROB2, EXP_X, FINAL_EXP   f                                    -> f'
//        LINE_DOUBLE                     T = (X, Y, Z) over Fp2               -> T' | line (c0, c1, c2)
//        LINE_ADD                        T | Q = (x, y) affine over Fp2       -> T' | line
//        G2_PREPARE                      Q                                    -> the 68 lines
//        MILLER                          the 68 lines | P = (x, y) over Fp    -> f
//        PAIR                            P | Q                                -> final_exponentiate(miller(prepare(Q), P)) | the 68 lines
//        IN_SUBGROUP_G1, IN_SUBGROUP_G2  P or Q                               -> 1 / 0
//   BN   LINE_AT                         lambda | xT | yT over Fq2 | P over Fq -> l(P)
//        MILLER_ATE, PAIR                P | Q                                -> miller_ate(Q, P), final_exponentiate of it
//        FINAL_EXP                       f                                    -> f'
//        IN_SUBGROUP_G2                  Q                                    -> 1 / 0
#include <cstring>
#include <initializer_list>

#include "bls_pairing.cuh"
#include "bn_pairing.cuh"

using namespace b200zk;

// a named namespace: the kernels' registration stub cannot tell an anonymous one from b200zk's
namespace pairing_conformance {

enum : int { T_BLS12_381 = 0, T_BN254 = 1 };
enum : int { FROB = 0, FROB2, EXP_X, FINAL_EXP, LINE_DOUBLE, LINE_ADD, G2_PREPARE, MILLER, PAIR, IN_SUBGROUP_G1, IN_SUBGROUP_G2,
             LINE_AT, MILLER_ATE, N_OPS };

template <class T> __device__ T ld(const uint32_t* p) { T t; memcpy(&t, p, sizeof(T)); return t; }
template <class T> __device__ void st(uint32_t* p, const T& t) { memcpy(p, &t, sizeof(T)); }
template <class T> __host__ __device__ constexpr uint32_t words() { return sizeof(T) / 4; }

// the prepared lines are read and written in place: plain 32-bit words, no padding
static_assert(alignof(BlsLine) == 4 && sizeof(BlsLine) == 3 * sizeof(F2), "BlsLine must be three packed Fp2 values");

__device__ inline uint64_t item() { return (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; }

__global__ void bls_kernel(int op, const uint32_t* in, uint32_t iw, uint32_t* out, uint32_t ow, uint64_t n) {
  const uint64_t i = item();
  if (i >= n) return;
  in += i * iw; out += i * ow;
  constexpr uint32_t WT = words<G2Proj>(), WP = words<Affine<Fp381>>(), WL = words<BlsLine>();
  switch (op) {
    case FROB: st(out, f12_frob(ld<F12>(in))); break;
    case FROB2: st(out, f12_frob2(ld<F12>(in))); break;
    case EXP_X: st(out, f12_exp_x(ld<F12>(in))); break;
    case FINAL_EXP: st(out, final_exponentiate(ld<F12>(in))); break;
    case LINE_DOUBLE: {
      Fp381 two_inv = fp381_half();  // 1/2 = (p + 1)/2 in Montgomery form, as g2_prepare makes it
      two_inv.v[0] += 1;
      two_inv = Fp381::to_mont(two_inv);
      G2Proj T = ld<G2Proj>(in);
      const BlsLine l = line_double(T, two_inv);
      st(out, T); st(out + WT, l);
      break;
    }
    case LINE_ADD: {
      G2Proj T = ld<G2Proj>(in);
      const BlsLine l = line_add(T, ld<Affine<F2>>(in + WT));
      st(out, T); st(out + WT, l);
      break;
    }
    case G2_PREPARE: g2_prepare(ld<Affine<F2>>(in), reinterpret_cast<BlsLine*>(out)); break;
    case MILLER: st(out, miller_prepared(reinterpret_cast<const BlsLine*>(in), ld<Affine<Fp381>>(in + kLines * WL))); break;
    case PAIR: {
      BlsLine* lines = reinterpret_cast<BlsLine*>(out + words<F12>());
      g2_prepare(ld<Affine<F2>>(in + WP), lines);
      st(out, final_exponentiate(miller_prepared(lines, ld<Affine<Fp381>>(in))));
      break;
    }
    case IN_SUBGROUP_G1: out[0] = in_subgroup<bls_r_limb>(ld<Affine<Fp381>>(in)) ? 1u : 0u; break;
    case IN_SUBGROUP_G2: out[0] = in_subgroup<bls_r_limb>(ld<Affine<F2>>(in)) ? 1u : 0u; break;
  }
}

__global__ void bn_kernel(int op, const uint32_t* in, uint32_t iw, uint32_t* out, uint32_t ow, uint64_t n) {
  const uint64_t i = item();
  if (i >= n) return;
  in += i * iw; out += i * ow;
  constexpr uint32_t W2 = words<Fq2>(), WP = words<Affine<Fq>>();
  switch (op) {
    case LINE_AT: st(out, line_at(ld<Fq2>(in), ld<Fq2>(in + W2), ld<Fq2>(in + 2 * W2), ld<Affine<Fq>>(in + 3 * W2))); break;
    case MILLER_ATE: st(out, miller_ate(ld<Affine<Fq2>>(in + WP), ld<Affine<Fq>>(in))); break;
    case FINAL_EXP: st(out, final_exponentiate(ld<Fq12>(in))); break;
    case PAIR: st(out, final_exponentiate(miller_ate(ld<Affine<Fq2>>(in + WP), ld<Affine<Fq>>(in)))); break;
    case IN_SUBGROUP_G2: out[0] = in_subgroup<FrCfg::mod>(ld<Affine<Fq2>>(in)) ? 1u : 0u; break;
  }
}

constexpr uint32_t bits(std::initializer_list<int> ops) {
  uint32_t m = 0;
  for (int o : ops) m |= 1u << o;
  return m;
}

uint32_t supported(int type) {
  switch (type) {
    case T_BLS12_381: return bits({FROB, FROB2, EXP_X, FINAL_EXP, LINE_DOUBLE, LINE_ADD, G2_PREPARE, MILLER, PAIR, IN_SUBGROUP_G1, IN_SUBGROUP_G2});
    case T_BN254: return bits({LINE_AT, MILLER_ATE, FINAL_EXP, PAIR, IN_SUBGROUP_G2});
  }
  return 0;
}

}  // namespace pairing_conformance

using namespace pairing_conformance;

// Runs op `op` of curve `type` on n items (device pointers, in_words / out_words 32-bit words per item) on the legacy
// default stream and waits for it.  0 on success, -1 for an unknown (type, op), else the CUDA error code.
extern "C" int b200zk_pairing_conformance_run(int type, int op, const uint32_t* in, uint32_t in_words, uint32_t* out, uint32_t out_words,
                                              uint64_t n) {
  if (op < 0 || op >= N_OPS || !((supported(type) >> op) & 1u)) return -1;
  if (n == 0) return 0;
  const uint32_t block = 32;
  const uint32_t grid = (uint32_t)((n + block - 1) / block);
  if (type == T_BLS12_381) bls_kernel<<<grid, block>>>(op, in, in_words, out, out_words, n);
  else bn_kernel<<<grid, block>>>(op, in, in_words, out, out_words, n);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  return (int)e;
}
