// field_conformance.cu -- test-only harness: every field and curve primitive of the product headers, one element per
// thread, so tests/test_gpu_field_conformance.py can compare each of them with Python integers at its limb edges; the
// pairing towers of tower.cuh op by op the same way.
// Not part of libb200zk.so; ethrex_b200/csrc/Makefile builds it with the product's own nvcc flags, so the code under
// test is generated exactly as the library's is.
//
// Layout: item i reads in[i * in_words ..] and writes out[i * out_words ..].  Field elements are their raw limbs
// (Montgomery or canonical, as the type keeps them; a quadratic extension is c0 then c1).  Operand k of a field op starts
// at word k * W, W the element's width in words.  One kernel per type, switching on the op at run time: FeBig's product
// is deliberately not inlined, and one instantiation per type keeps the compile time of this file bounded.
#include <cstring>
#include <initializer_list>
#include <type_traits>

#include "field.cuh"
#include "curve.cuh"
#include "bls381.cuh"
#include "common.cuh"
#include "bls12.cuh"
#include "tower.cuh"
#include "secp256k1.cuh"

using namespace b200zk;

namespace {

// type ids
enum : int { T_FQ = 0, T_FR = 1, T_FQ2 = 2, T_FP381 = 3, T_FR381 = 4, T_FP2_381 = 5, T_SECP_FP = 6, T_SECP_FN = 7, T_BYTES = 8,
             T_BN_G1 = 10, T_BN_G2 = 11, T_BLS_G1 = 12, T_BLS_G2 = 13, T_SECP_G = 14,
             T_BN_FP6 = 15, T_BN_FP12 = 16, T_BLS_FP6 = 17, T_BLS_FP12 = 18 };
// field op ids
enum : int { ADD = 0, SUB, NEG, DBL, MUL, SQR, MUL2_ADD, MUL2_SUB, MUL4_ADD, TO_MONT, FROM_MONT, INV, POW, LESS, SQRT, CONJ,
             MUL_XI, SCALE, N_FIELD_OPS };
// byte-format op ids (T_BYTES)
enum : int { LOAD_BE48 = 0, LOAD_BE48_MASKED, STORE_BE48, LOAD_FP64, LOAD_BE32, LOAD_BE256, STORE_BE256, N_BYTE_OPS };
// curve op ids: XYZZ points are x | y | zz | zzz, affine points x | y, scalars 8 little-endian limbs
enum : int { C_ADD = 0, C_ADD_MIXED, C_DBL, C_MDBL, C_TO_AFFINE, C_SCALAR_MUL, C_ON_CURVE, N_CURVE_OPS };
// tower op ids (tower.cuh): the sparse products' F2 operands follow the tower element
enum : int { X_ZERO = 0, X_ONE, X_ADD, X_SUB, X_NEG, X_MUL_V, X_MUL, X_SQR, X_CONJ, X_INV, X_IS_ONE, X_MUL_01, X_MUL_1, X_MUL_014,
             N_TOWER_OPS };

template <class T> __device__ T ld(const uint32_t* p) { T t; memcpy(&t, p, sizeof(T)); return t; }
template <class T> __device__ void st(uint32_t* p, const T& t) { memcpy(p, &t, sizeof(T)); }
template <class T> __host__ __device__ constexpr uint32_t words() { return sizeof(T) / 4; }

__device__ inline uint64_t item() { return (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; }

// BN254 Fq, Fr
template <class F> __global__ void fe_kernel(int op, const uint32_t* in, uint32_t iw, uint32_t* out, uint32_t ow, uint64_t n) {
  const uint64_t i = item();
  if (i >= n) return;
  in += i * iw; out += i * ow;
  constexpr uint32_t W = words<F>();
  auto x = [&](int k) { return ld<F>(in + k * W); };
  switch (op) {
    case ADD: st(out, F::add(x(0), x(1))); break;
    case SUB: st(out, F::sub(x(0), x(1))); break;
    case NEG: st(out, F::neg(x(0))); break;
    case DBL: st(out, F::dbl(x(0))); break;
    case MUL: st(out, F::mul(x(0), x(1))); break;
    case SQR: st(out, F::sqr(x(0))); break;
    case MUL2_ADD: st(out, F::mul2_add(x(0), x(1), x(2), x(3))); break;
    case MUL2_SUB: st(out, F::mul2_sub(x(0), x(1), x(2), x(3))); break;
    case MUL4_ADD: st(out, F::mul4_add(x(0), x(1), x(2), x(3), x(4), x(5), x(6), x(7))); break;
    case TO_MONT: st(out, F::to_mont(x(0))); break;
    case FROM_MONT: st(out, F::from_mont(x(0))); break;
    case INV: st(out, F::inv(x(0))); break;
    case POW: st(out, F::pow(x(0), in + W)); break;
  }
}

__global__ void fq2_kernel(int op, const uint32_t* in, uint32_t iw, uint32_t* out, uint32_t ow, uint64_t n) {
  const uint64_t i = item();
  if (i >= n) return;
  in += i * iw; out += i * ow;
  constexpr uint32_t W = words<Fq2>();
  auto x = [&](int k) { return ld<Fq2>(in + k * W); };
  switch (op) {
    case ADD: st(out, Fq2::add(x(0), x(1))); break;
    case SUB: st(out, Fq2::sub(x(0), x(1))); break;
    case NEG: st(out, Fq2::neg(x(0))); break;
    case DBL: st(out, Fq2::dbl(x(0))); break;
    case MUL: st(out, Fq2::mul(x(0), x(1))); break;
    case SQR: st(out, Fq2::sqr(x(0))); break;
    case MUL2_SUB: st(out, Fq2::mul2_sub(x(0), x(1), x(2), x(3))); break;
    case INV: st(out, Fq2::inv(x(0))); break;
    case MUL_XI: st(out, Fq2::mul_xi(x(0))); break;
  }
}

// BLS12-381 Fp, Fr (FeBig); sqrt_candidate exists for Fp only
template <class F> __global__ void big_kernel(int op, const uint32_t* in, uint32_t iw, uint32_t* out, uint32_t ow, uint64_t n) {
  const uint64_t i = item();
  if (i >= n) return;
  in += i * iw; out += i * ow;
  constexpr uint32_t W = words<F>();
  auto x = [&](int k) { return ld<F>(in + k * W); };
  switch (op) {
    case ADD: st(out, F::add(x(0), x(1))); break;
    case SUB: st(out, F::sub(x(0), x(1))); break;
    case NEG: st(out, F::neg(x(0))); break;
    case DBL: st(out, F::dbl(x(0))); break;
    case MUL: st(out, F::mul(x(0), x(1))); break;
    case SQR: st(out, F::sqr(x(0))); break;
    case MUL2_SUB: st(out, F::mul2_sub(x(0), x(1), x(2), x(3))); break;
    case TO_MONT: st(out, F::to_mont(x(0))); break;
    case FROM_MONT: st(out, F::from_mont(x(0))); break;
    case INV: st(out, F::inv(x(0))); break;
    case POW: st(out, F::pow(x(0), in + W)); break;
    case LESS: out[0] = F::less(x(0), x(1)) ? 1u : 0u; break;
    case SQRT:
      if constexpr (std::is_same<F, Fp381>::value) st(out, F::sqrt_candidate(x(0)));
      break;
  }
}

__global__ void fp2_381_kernel(int op, const uint32_t* in, uint32_t iw, uint32_t* out, uint32_t ow, uint64_t n) {
  const uint64_t i = item();
  if (i >= n) return;
  in += i * iw; out += i * ow;
  constexpr uint32_t W = words<Fp2_381>();
  auto x = [&](int k) { return ld<Fp2_381>(in + k * W); };
  switch (op) {
    case ADD: st(out, Fp2_381::add(x(0), x(1))); break;
    case SUB: st(out, Fp2_381::sub(x(0), x(1))); break;
    case NEG: st(out, Fp2_381::neg(x(0))); break;
    case DBL: st(out, Fp2_381::dbl(x(0))); break;
    case CONJ: st(out, Fp2_381::conj(x(0))); break;
    case MUL: st(out, Fp2_381::mul(x(0), x(1))); break;
    case SQR: st(out, Fp2_381::sqr(x(0))); break;
    case MUL_XI: st(out, Fp2_381::mul_xi(x(0))); break;
    case SCALE: st(out, Fp2_381::scale(x(0), ld<Fp381>(in + W))); break;  // k: the first 12 words of operand 1
    case MUL2_SUB: st(out, Fp2_381::mul2_sub(x(0), x(1), x(2), x(3))); break;
    case INV: st(out, Fp2_381::inv(x(0))); break;
    case POW: st(out, Fp2_381::pow(x(0), in + W)); break;  // e: 12 limbs
    case SQRT: st(out, Fp2_381::sqrt_candidate(x(0))); break;
  }
}

// secp256k1 base field (canonical) and scalar field (Montgomery); SQRT writes the root, then 1 / 0 for "a is a square"
__global__ void secp_kernel(int type, int op, const uint32_t* in, uint32_t iw, uint32_t* out, uint32_t ow, uint64_t n) {
  const uint64_t i = item();
  if (i >= n) return;
  in += i * iw; out += i * ow;
  if (type == T_SECP_FP) {
    auto x = [&](int k) { return ld<SecpFp>(in + k * 8); };
    switch (op) {
      case ADD: st(out, SecpFp::add(x(0), x(1))); break;
      case SUB: st(out, SecpFp::sub(x(0), x(1))); break;
      case NEG: st(out, SecpFp::neg(x(0))); break;
      case DBL: st(out, SecpFp::dbl(x(0))); break;
      case MUL: st(out, SecpFp::mul(x(0), x(1))); break;
      case SQR: st(out, SecpFp::sqr(x(0))); break;
      case MUL2_SUB: st(out, SecpFp::mul2_sub(x(0), x(1), x(2), x(3))); break;
      case INV: st(out, SecpFp::inv(x(0))); break;
      case POW: st(out, SecpFp::pow(x(0), in + 8)); break;
      case SQRT: { SecpFp r; const bool ok = SecpFp::sqrt(x(0), &r); st(out, r); out[8] = ok ? 1u : 0u; break; }
    }
  } else {
    auto x = [&](int k) { return ld<SecpFn>(in + k * 8); };
    switch (op) {
      case NEG: st(out, SecpFn::neg(x(0))); break;
      case MUL: st(out, SecpFn::mul(x(0), x(1))); break;
      case TO_MONT: st(out, SecpFn::from_canonical(in)); break;
      case FROM_MONT: x(0).to_canonical(out); break;
      case INV: st(out, SecpFn::inv(x(0))); break;
    }
  }
}

// byte formats: byte strings travel as words in memory order
__global__ void bytes_kernel(int op, const uint32_t* in, uint32_t iw, uint32_t* out, uint32_t ow, uint64_t n) {
  const uint64_t i = item();
  if (i >= n) return;
  in += i * iw; out += i * ow;
  const uint8_t* b = reinterpret_cast<const uint8_t*>(in);
  switch (op) {
    case LOAD_BE48: st(out, load_be48(b, 0xffffffffu)); break;
    case LOAD_BE48_MASKED: st(out, load_be48(b, 0x1fffffffu)); break;
    case STORE_BE48: store_be48(reinterpret_cast<uint8_t*>(out), ld<Fp381>(in)); break;
    case LOAD_FP64: { Fp381 v; const bool ok = load_fp64(b, &v); st(out, v); out[12] = ok ? 1u : 0u; break; }
    case LOAD_BE32: st(out, load_be32(b)); break;
    case LOAD_BE256: secp::load_be256(out, b); break;
    case STORE_BE256: secp::store_be256(reinterpret_cast<uint8_t*>(out), in); break;
  }
}

template <class F> __global__ void curve_kernel(int op, const uint32_t* in, uint32_t iw, uint32_t* out, uint32_t ow, uint64_t n) {
  const uint64_t i = item();
  if (i >= n) return;
  in += i * iw; out += i * ow;
  constexpr uint32_t W = words<F>();
  switch (op) {
    case C_ADD: { XYZZ<F> a = ld<XYZZ<F>>(in); xyzz_add(a, ld<XYZZ<F>>(in + 4 * W)); st(out, a); break; }
    case C_ADD_MIXED: { XYZZ<F> a = ld<XYZZ<F>>(in); xyzz_add_mixed(a, ld<F>(in + 4 * W), ld<F>(in + 5 * W)); st(out, a); break; }
    case C_DBL: st(out, xyzz_dbl(ld<XYZZ<F>>(in))); break;
    case C_MDBL: st(out, xyzz_mdbl(ld<F>(in), ld<F>(in + W))); break;
    case C_TO_AFFINE: st(out, xyzz_to_affine(ld<XYZZ<F>>(in))); break;
    case C_SCALAR_MUL: st(out, xyzz_scalar_mul(in + 2 * W, ld<Affine<F>>(in))); break;
    case C_ON_CURVE: out[0] = affine_on_curve(ld<Affine<F>>(in)) ? 1u : 0u; break;
  }
}

// Fp6<F2> and Fp12<F2>; IS_ONE writes 1 / 0
template <class F2> __global__ void fp6_kernel(int op, const uint32_t* in, uint32_t iw, uint32_t* out, uint32_t ow, uint64_t n) {
  typedef Fp6<F2> E;
  const uint64_t i = item();
  if (i >= n) return;
  in += i * iw; out += i * ow;
  constexpr uint32_t W = words<E>();
  auto x = [&](int k) { return ld<E>(in + k * W); };
  auto y = [&](int k) { return ld<F2>(in + W + k * words<F2>()); };
  switch (op) {
    case X_ZERO: st(out, E::zero()); break;
    case X_ONE: st(out, E::one()); break;
    case X_ADD: st(out, E::add(x(0), x(1))); break;
    case X_SUB: st(out, E::sub(x(0), x(1))); break;
    case X_NEG: st(out, E::neg(x(0))); break;
    case X_MUL_V: st(out, E::mul_v(x(0))); break;
    case X_MUL: st(out, E::mul(x(0), x(1))); break;
    case X_INV: st(out, E::inv(x(0))); break;
    case X_MUL_01: st(out, E::mul_01(x(0), y(0), y(1))); break;
    case X_MUL_1: st(out, E::mul_1(x(0), y(0))); break;
  }
}

template <class F2> __global__ void fp12_kernel(int op, const uint32_t* in, uint32_t iw, uint32_t* out, uint32_t ow, uint64_t n) {
  typedef Fp12<F2> E;
  const uint64_t i = item();
  if (i >= n) return;
  in += i * iw; out += i * ow;
  constexpr uint32_t W = words<E>();
  auto x = [&](int k) { return ld<E>(in + k * W); };
  auto y = [&](int k) { return ld<F2>(in + W + k * words<F2>()); };
  switch (op) {
    case X_ONE: st(out, E::one()); break;
    case X_MUL: st(out, E::mul(x(0), x(1))); break;
    case X_SQR: st(out, E::sqr(x(0))); break;
    case X_CONJ: st(out, E::conj(x(0))); break;
    case X_INV: st(out, E::inv(x(0))); break;
    case X_IS_ONE: out[0] = E::is_one(x(0)) ? 1u : 0u; break;
    case X_MUL_014: st(out, E::mul_014(x(0), y(0), y(1), y(2))); break;
  }
}

constexpr uint32_t bits(std::initializer_list<int> ops) {
  uint32_t m = 0;
  for (int o : ops) m |= 1u << o;
  return m;
}

// the ops each type implements
uint32_t supported(int type) {
  switch (type) {
    case T_FQ: case T_FR:
      return bits({ADD, SUB, NEG, DBL, MUL, SQR, MUL2_ADD, MUL2_SUB, MUL4_ADD, TO_MONT, FROM_MONT, INV, POW});
    case T_FQ2: return bits({ADD, SUB, NEG, DBL, MUL, SQR, MUL2_SUB, INV, MUL_XI});
    case T_FP381: return bits({ADD, SUB, NEG, DBL, MUL, SQR, MUL2_SUB, TO_MONT, FROM_MONT, INV, POW, LESS, SQRT});
    case T_FR381: return bits({ADD, SUB, NEG, DBL, MUL, SQR, MUL2_SUB, TO_MONT, FROM_MONT, INV, POW, LESS});
    case T_FP2_381: return bits({ADD, SUB, NEG, DBL, CONJ, MUL, SQR, MUL_XI, SCALE, MUL2_SUB, INV, POW, SQRT});
    case T_SECP_FP: return bits({ADD, SUB, NEG, DBL, MUL, SQR, MUL2_SUB, INV, POW, SQRT});
    case T_SECP_FN: return bits({NEG, MUL, TO_MONT, FROM_MONT, INV});
    case T_BYTES: return (1u << N_BYTE_OPS) - 1;
    case T_BN_G1: case T_BN_G2: case T_BLS_G1: case T_BLS_G2: case T_SECP_G: return (1u << N_CURVE_OPS) - 1;
    case T_BN_FP6: case T_BLS_FP6: return bits({X_ZERO, X_ONE, X_ADD, X_SUB, X_NEG, X_MUL_V, X_MUL, X_INV, X_MUL_01, X_MUL_1});
    case T_BN_FP12: case T_BLS_FP12: return bits({X_ONE, X_MUL, X_SQR, X_CONJ, X_INV, X_IS_ONE, X_MUL_014});
  }
  return 0;
}

}  // namespace

// Runs op `op` of type `type` on n items (device pointers, in_words / out_words 32-bit words per item) on the legacy
// default stream and waits for it.  0 on success, -1 for an unknown (type, op), else the CUDA error code.
extern "C" int b200zk_conformance_run(int type, int op, const uint32_t* in, uint32_t in_words, uint32_t* out, uint32_t out_words,
                                      uint64_t n) {
  if (op < 0 || op >= 32 || !((supported(type) >> op) & 1u)) return -1;
  if (n == 0) return 0;
  const uint32_t block = 128;
  const uint32_t grid = (uint32_t)((n + block - 1) / block);
  switch (type) {
    case T_FQ: fe_kernel<Fq><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_FR: fe_kernel<Fr><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_FQ2: fq2_kernel<<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_FP381: big_kernel<Fp381><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_FR381: big_kernel<Fr381><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_FP2_381: fp2_381_kernel<<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_SECP_FP: case T_SECP_FN: secp_kernel<<<grid, block>>>(type, op, in, in_words, out, out_words, n); break;
    case T_BYTES: bytes_kernel<<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_BN_G1: curve_kernel<Fq><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_BN_G2: curve_kernel<Fq2><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_BLS_G1: curve_kernel<Fp381><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_BLS_G2: curve_kernel<Fp2_381><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_SECP_G: curve_kernel<SecpFp><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_BN_FP6: fp6_kernel<Fq2><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_BN_FP12: fp12_kernel<Fq2><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_BLS_FP6: fp6_kernel<Fp2_381><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
    case T_BLS_FP12: fp12_kernel<Fp2_381><<<grid, block>>>(op, in, in_words, out, out_words, n); break;
  }
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  return (int)e;
}
