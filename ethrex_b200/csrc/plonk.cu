// plonk.cu -- snarkjs 0.7 PLONK from circom artifacts: a .zkey loaded once into HBM, each .wtns witness proved in one call
// (b200zk_plonk_zkey_*; formats in include/b200zk.h, parser in zkey_parse.cpp).
//
//   load    parse (host) -> PTau as a resident handle (window tables on request), every point on its curve -> the
//           coefficients of Qm Ql Qr Qo Qc S1 S2 S3 -> S1..S3 on the domain (NTT n) and the 8 polynomials and L1 on the
//           coset 5 <w_4n> (coset NTT 4n) -> the additions grouped by dependency level (host)
//   prove   round 1  witness range check, additions (plonk_additions, one launch per level), a b c through the maps
//                    (plonk_gather), iNTT n, blinding (plonk_blind), three MSMs; transcript -> beta, gamma
//           round 2  num / den per row with a batch inversion (plonk_perm_ratio), Z = their prefix product (the affine
//                    scan below, which also checks the full product), iNTT n, blinding, MSM; transcript -> alpha
//           round 3  A B C Z and PI on the coset, T = N / Z_H pointwise (plonk_quotient), coset iNTT 4n, the gate check
//                    on T's top coefficients, T1 T2 T3 (plonk_split), three MSMs; transcript -> xi
//           round 4  A B C S1 S2 at xi and Z at xi w as block reductions (plonk_eval), L1(xi), PI(xi), Z_H(xi)
//                    (plonk_eval_finish); transcript -> v1..v5 and the linearisation's scalars
//           round 5  the numerators of Wxi and Wxiw (plonk_linearise), the divisions by (X - xi) and (X - xi w) as the
//                    affine scan, two MSMs
// Everything runs on one stream; the challenges never leave the device (plonk_transcript reads the encoded commitments
// the MSMs left there), and the proof, the witness check and the two satisfaction flags come back in one copy.
//
// The affine scan: x_0 given, x_(k+1) = a_k x_k + b_k, every x_k written out.  Z is a_k = num_k / den_k, b = 0, x_0 = 1
// (x_n is the full product, which must be 1); q = p / (X - x0) is a = x0, b_k = p_(m-1-k), x_0 = 0 written from the top
// (x_k = q_(m-1-k)).  Each thread composes the affine maps of one chunk; one CTA turns the chunk maps into each chunk's
// incoming x; each thread then writes its chunk.
#include "common.cuh"
#include "keccak.cuh"
#include "zkey_parse.h"

#include <algorithm>
#include <cstring>
#include <vector>

namespace b200zk {

namespace {

struct Limbs8Arg { uint32_t v[8]; };

// Fr slots of PlonkEntry::consts (Montgomery); the verifying key's bytes follow at kVkOff
enum { kCK1 = 0, kCK2, kCW, kCWinv, kCW4, kCNinv, kCGen, kCZhInv /* 4 slots */, kCSlots = kCZhInv + 4 };
constexpr size_t kVkOff = 32 * 16;
constexpr size_t kVkBytes = 736;
// Fr slots of a prove's challenge block (Montgomery)
enum {
  kBeta = 0, kGamma, kAlpha, kXi, kV1, kV2, kV3, kV4, kV5,
  kEa, kEb, kEc, kEs1, kEs2, kEzw,  // the six evaluations (plonk_eval_finish)
  kXiW, kXin, kZh, kL1, kPi,        // xi w, xi^n, Z_H(xi), L1(xi), PI(xi)
  kRab, kRz, kRs3, kRc0,            // linearisation: eval_a eval_b, Z's scalar, -S3's scalar, the constant of Wxi's numerator
  kChSlots = 32
};
constexpr uint32_t kRatioChunk = 32;  // rows per thread of plonk_perm_ratio (one inversion each)
constexpr uint32_t kEvalChunk = 16;   // coefficients per thread of plonk_eval
constexpr uint32_t kQuotChunk = 8;    // coset points per thread of plonk_quotient (one power each)

B2_D Fr pow_u64(Fr a, uint64_t e) {
  Fr r = Fr::one();
  for (; e; e >>= 1) { if (e & 1) r = Fr::mul(r, a); a = Fr::sqr(a); }
  return r;
}
B2_D Fr ldc(const void* p, int slot) { return load_fe<Fr>(p, slot); }
// 32-byte big-endian canonical value of a Montgomery element
template <class F> B2_D void put_be(uint8_t* out, const F& mont) {
  const F v = F::from_mont(mont);
  for (int k = 0; k < 8; ++k) {
    const uint32_t limb = v.v[7 - k];
    out[4 * k] = (uint8_t)(limb >> 24); out[4 * k + 1] = (uint8_t)(limb >> 16); out[4 * k + 2] = (uint8_t)(limb >> 8); out[4 * k + 3] = (uint8_t)limb;
  }
}
B2_D Fr blind_at(const void* blind, int k) { return Fr::to_mont(load_fe<Fr>(blind, k - 1)); }  // b_k (1-based), canonical in memory

// ---- load -----------------------------------------------------------------------------------------------------------
// the constants: w_4n = root^(2^(26 - log_n)) from the preset-0 2^28-th root (canonical), w_n, 1/w_n, 1/n, 5, and
// 1 / Z_H on the coset's four classes, 1 / (5^n w_4^j - 1); k1 and k2 are already in their slots.  Then the verifying key:
// the 8 G1 commitments and X_2 (EIP-196/197) and k1, k2, w_n as big-endian canonical values
__global__ void plonk_consts(Limbs8Arg root, uint32_t log_n, const void* hdr_points, void* consts) {
  if (blockIdx.x || threadIdx.x) return;
  Fr g;
  for (int k = 0; k < 8; ++k) g.v[k] = root.v[k];
  g = Fr::to_mont(g);
  for (uint32_t i = log_n + 2; i < 28; ++i) g = Fr::sqr(g);
  const Fr w4 = g, w = Fr::sqr(Fr::sqr(w4));
  const uint64_t n = 1ull << log_n;
  Fr nn = Fr::zero();
  nn.v[0] = (uint32_t)n;
  nn.v[1] = (uint32_t)(n >> 32);
  Fr five = Fr::zero();
  five.v[0] = 5;
  five = Fr::to_mont(five);
  store_fe<Fr>(consts, kCW, w);
  store_fe<Fr>(consts, kCWinv, Fr::inv(w));
  store_fe<Fr>(consts, kCW4, w4);
  store_fe<Fr>(consts, kCNinv, Fr::inv(Fr::to_mont(nn)));
  store_fe<Fr>(consts, kCGen, five);
  const Fr w_4 = pow_u64(w4, n), gn = pow_u64(five, n);
  Fr c = gn;
  for (int j = 0; j < 4; ++j) { store_fe<Fr>(consts, kCZhInv + j, Fr::inv(Fr::sub(c, Fr::one()))); c = Fr::mul(c, w_4); }
  uint8_t* vk = (uint8_t*)consts + kVkOff;
  for (int k = 0; k < 16; ++k) put_be<Fq>(vk + 32 * k, load_fe<Fq>(hdr_points, k));
  const int kG2Order[4] = {1, 0, 3, 2};  // x_im | x_re | y_im | y_re from x.c0 x.c1 y.c0 y.c1
  for (int k = 0; k < 4; ++k) put_be<Fq>(vk + 512 + 32 * k, load_fe<Fq>(hdr_points, 16 + kG2Order[k]));
  put_be<Fr>(vk + 640, ldc(consts, kCK1));
  put_be<Fr>(vk + 672, ldc(consts, kCK2));
  put_be<Fr>(vk + 704, w);
}

// out[i] = the Fr value of slot `slot` of consts, i < n (L1's coefficients, all 1/n)
__global__ void __launch_bounds__(256) plonk_fill(void* out, size_t n, const void* consts, int slot) {
  const Fr v = ldc(consts, slot);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) store_fe<Fr>(out, i, v);
}

// ---- prove: round 1 ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) plonk_range_check(const void* wit, size_t n, unsigned long long* bad) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    Fr v = load_fe_nc<Fr>(wit, i), m = Fr::modulus(), t;
    if (!detail::sub8(t.v, v.v, m.v)) atomicMin(bad, (unsigned long long)i);
  }
}

// additions [begin, end) of one level: w[dst] = f1 w[s1] + f2 w[s2] (f Montgomery, w canonical: the products are canonical)
__global__ void __launch_bounds__(256) plonk_additions(const uint4* rec, const void* f1, const void* f2, uint32_t begin, uint32_t end, void* wit) {
  const uint32_t i = begin + blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= end) return;
  const uint4 r = rec[i];
  const Fr v = Fr::add(Fr::mul(load_fe<Fr>(f1, i), load_fe<Fr>(wit, r.y)), Fr::mul(load_fe<Fr>(f2, i), load_fe<Fr>(wit, r.z)));
  store_fe<Fr>(wit, r.x, v);
}

// a, b, c on the domain (Montgomery): w through the maps for rows < nConstraints, zero after; PI's values -a_i on the
// public rows into pi (when given)
__global__ void __launch_bounds__(256) plonk_gather(const uint32_t* maps, uint32_t n_constraints, uint32_t n_public, size_t n, const void* wit, void* abc, void* pi) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    for (int k = 0; k < 3; ++k) {
      const Fr v = i < n_constraints ? Fr::to_mont(load_fe<Fr>(wit, __ldg(maps + (size_t)k * n_constraints + i))) : Fr::zero();
      store_fe<Fr>(abc, (size_t)k * n + i, v);
      if (k == 0 && pi && i < n_public) store_fe<Fr>(pi, i, Fr::neg(v));
    }
  }
}

// snarkjs's blindCoefficients: coef += sum_j f_j (X^(n+j) - X^j), f_j = b_(idx[j]); coef[n..n+count) must be zero before
__global__ void plonk_blind(void* coef, size_t n, const void* blind, int count, int i0, int i1, int i2) {
  if (blockIdx.x || threadIdx.x) return;
  const int idx[3] = {i0, i1, i2};
  for (int j = 0; j < count; ++j) {
    const Fr f = blind_at(blind, idx[j]);
    store_fe<Fr>(coef, n + j, Fr::add(load_fe<Fr>(coef, n + j), f));
    store_fe<Fr>(coef, j, Fr::sub(load_fe<Fr>(coef, j), f));
  }
}

// ---- the transcript ---------------------------------------------------------------------------------------------------
// keccak256 of buf[0, len) mod r, Montgomery
B2_D Fr challenge(const uint8_t* buf, size_t len) {
  uint8_t h[32];
  keccak256(buf, len, h);
  Fr v, m = Fr::modulus(), t;
  for (int k = 0; k < 8; ++k) v.v[k] = (uint32_t)h[31 - 4 * k] | (uint32_t)h[30 - 4 * k] << 8 | (uint32_t)h[29 - 4 * k] << 16 | (uint32_t)h[28 - 4 * k] << 24;
  while (!detail::sub8(t.v, v.v, m.v)) v = t;  // 2^256 < 6 r
  return Fr::to_mont(v);
}
B2_D size_t put_point(uint8_t* buf, size_t off, const uint8_t* enc) { for (int k = 0; k < 64; ++k) buf[off + k] = enc[k]; return off + 64; }
B2_D size_t put_fr(uint8_t* buf, size_t off, const Fr& v) { put_be<Fr>(buf + off, v); return off + 32; }

// One thread.  enc: the commitments, 128 bytes apart (A B C Z T1 T2 T3 Wxi Wxiw, BE x | y as msm_encode leaves them);
// ev_out: the proof's six evaluations (round 3 writes them).
//   round 0: beta = H(vk's 8 points, public inputs, A, B, C), gamma = H(beta)      round 1: alpha = H(beta, gamma, Z)
//   round 2: xi = H(alpha, T1, T2, T3)       round 3: v1 = H(xi, the evaluations), v2..v5, then the linearisation's scalars
__global__ void plonk_transcript(int round, const void* consts, const void* a_h, uint32_t n_public, const uint8_t* enc, void* ch, uint8_t* buf, uint8_t* ev_out) {
  if (blockIdx.x || threadIdx.x) return;
  size_t off = 0;
  if (round == 0) {
    const uint8_t* vk = (const uint8_t*)consts + kVkOff;
    for (int k = 0; k < 512; ++k) buf[k] = vk[k];
    off = 512;
    for (uint32_t i = 0; i < n_public; ++i) off = put_fr(buf, off, load_fe<Fr>(a_h, i));
    for (int k = 0; k < 3; ++k) off = put_point(buf, off, enc + 128 * k);
    const Fr beta = challenge(buf, off);
    store_fe<Fr>(ch, kBeta, beta);
    put_fr(buf, 0, beta);
    store_fe<Fr>(ch, kGamma, challenge(buf, 32));
  } else if (round == 1) {
    off = put_fr(buf, off, ldc(ch, kBeta));
    off = put_fr(buf, off, ldc(ch, kGamma));
    off = put_point(buf, off, enc + 128 * 3);
    store_fe<Fr>(ch, kAlpha, challenge(buf, off));
  } else if (round == 2) {
    off = put_fr(buf, off, ldc(ch, kAlpha));
    for (int k = 4; k < 7; ++k) off = put_point(buf, off, enc + 128 * k);
    store_fe<Fr>(ch, kXi, challenge(buf, off));
  } else {
    off = put_fr(buf, off, ldc(ch, kXi));
    for (int k = 0; k < 6; ++k) { put_fr(ev_out, 32 * k, ldc(ch, kEa + k)); off = put_fr(buf, off, ldc(ch, kEa + k)); }
    const Fr v1 = challenge(buf, off);
    Fr v = v1;
    for (int k = 0; k < 5; ++k) { store_fe<Fr>(ch, kV1 + k, v); v = Fr::mul(v, v1); }
    // R = eval_a eval_b Qm + eval_a Ql + eval_b Qr + eval_c Qo + Qc + (d2a + alpha^2 L1(xi)) Z - d3 S3
    //     - Z_H(xi) (T1 + xi^n T2 + xi^2n T3) + r0 (snarkjs 0.7 plonk_verify.js calculateD and calculateR0)
    const Fr beta = ldc(ch, kBeta), gamma = ldc(ch, kGamma), alpha = ldc(ch, kAlpha), xi = ldc(ch, kXi);
    const Fr ea = ldc(ch, kEa), eb = ldc(ch, kEb), ec = ldc(ch, kEc), es1 = ldc(ch, kEs1), es2 = ldc(ch, kEs2), ezw = ldc(ch, kEzw);
    const Fr a2 = Fr::sqr(alpha), l1 = ldc(ch, kL1), bxi = Fr::mul(beta, xi);
    const Fr d2a = Fr::mul(Fr::mul(Fr::mul(alpha, Fr::add(Fr::add(ea, bxi), gamma)), Fr::add(Fr::add(eb, Fr::mul(bxi, ldc(consts, kCK1))), gamma)),
                           Fr::add(Fr::add(ec, Fr::mul(bxi, ldc(consts, kCK2))), gamma));
    const Fr e3a = Fr::add(Fr::add(ea, Fr::mul(beta, es1)), gamma), e3b = Fr::add(Fr::add(eb, Fr::mul(beta, es2)), gamma);
    const Fr e3 = Fr::mul(Fr::mul(alpha, ezw), Fr::mul(e3a, e3b));
    store_fe<Fr>(ch, kRab, Fr::mul(ea, eb));
    store_fe<Fr>(ch, kRz, Fr::add(d2a, Fr::mul(l1, a2)));
    store_fe<Fr>(ch, kRs3, Fr::mul(e3, beta));
    Fr c0 = Fr::sub(Fr::sub(ldc(ch, kPi), Fr::mul(l1, a2)), Fr::mul(e3, Fr::add(ec, gamma)));  // r0
    const Fr evs[5] = {ea, eb, ec, es1, es2};
    for (int k = 0; k < 5; ++k) c0 = Fr::sub(c0, Fr::mul(ldc(ch, kV1 + k), evs[k]));
    store_fe<Fr>(ch, kRc0, c0);
  }
}

// ---- round 2: the permutation argument ---------------------------------------------------------------------------------
// ratio[i] = num_i / den_i for the rows of one chunk, one inversion per chunk (Montgomery's trick):
//   num_i = (a + beta w^i + gamma)(b + beta k1 w^i + gamma)(c + beta k2 w^i + gamma)
//   den_i = (a + beta S1 + gamma)(b + beta S2 + gamma)(c + beta S3 + gamma)
struct PermTerms { Fr num, den; };
B2_D PermTerms perm_terms(const void* abc, const void* sig, size_t n, size_t i, const Fr& x, const Fr& beta, const Fr& gamma, const Fr& k1, const Fr& k2) {
  const Fr a = load_fe<Fr>(abc, i), b = load_fe<Fr>(abc, n + i), c = load_fe<Fr>(abc, 2 * n + i);
  const Fr bx = Fr::mul(beta, x);
  PermTerms t;
  t.num = Fr::mul(Fr::mul(Fr::add(Fr::add(a, bx), gamma), Fr::add(Fr::add(b, Fr::mul(bx, k1)), gamma)), Fr::add(Fr::add(c, Fr::mul(bx, k2)), gamma));
  t.den = Fr::mul(Fr::mul(Fr::add(Fr::add(a, Fr::mul(beta, load_fe_nc<Fr>(sig, i))), gamma), Fr::add(Fr::add(b, Fr::mul(beta, load_fe_nc<Fr>(sig, n + i))), gamma)),
                  Fr::add(Fr::add(c, Fr::mul(beta, load_fe_nc<Fr>(sig, 2 * n + i))), gamma));
  return t;
}
__global__ void __launch_bounds__(128) plonk_perm_ratio(const void* abc, const void* sig, size_t n, const void* consts, const void* ch, void* ratio) {
  const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x, r0 = t * kRatioChunk;
  if (r0 >= n) return;
  const size_t r1 = n < r0 + kRatioChunk ? n : r0 + kRatioChunk;
  const Fr beta = ldc(ch, kBeta), gamma = ldc(ch, kGamma), k1 = ldc(consts, kCK1), k2 = ldc(consts, kCK2), w = ldc(consts, kCW);
  Fr x = pow_u64(w, r0), acc = Fr::one();
  for (size_t i = r0; i < r1; ++i) {  // prefix products of den
    acc = Fr::mul(acc, perm_terms(abc, sig, n, i, x, beta, gamma, k1, k2).den);
    store_fe<Fr>(ratio, i, acc);
    if (i + 1 < r1) x = Fr::mul(x, w);
  }
  Fr inv = Fr::inv(acc);
  const Fr winv = ldc(consts, kCWinv);
  for (size_t i = r1; i-- > r0;) {
    const PermTerms pt = perm_terms(abc, sig, n, i, x, beta, gamma, k1, k2);
    const Fr dinv = i > r0 ? Fr::mul(inv, load_fe<Fr>(ratio, i - 1)) : inv;
    inv = Fr::mul(inv, pt.den);
    store_fe<Fr>(ratio, i, Fr::mul(pt.num, dinv));
    x = Fr::mul(x, winv);
  }
}

// ---- the affine scan ---------------------------------------------------------------------------------------------------
// DIV = false: a_k = arr[k], b_k = 0, out[k] = x_k.   DIV = true: a_k = *a_const, b_k = arr[m - 1 - k], out[m - 1 - k] = x_k.
// out may be arr (each element is read before it is written).
template <bool DIV> B2_D Fr scan_a(const void* arr, const Fr& ac, size_t k) { return DIV ? ac : load_fe<Fr>(arr, k); }
template <bool DIV> B2_D Fr scan_b(const void* arr, size_t m, size_t k) { return DIV ? load_fe<Fr>(arr, m - 1 - k) : Fr::zero(); }

template <bool DIV>
__global__ void __launch_bounds__(256) plonk_scan_compose(const void* arr, const void* a_const, size_t m, uint32_t chunk, void* comp) {
  const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x, k0 = t * chunk;
  if (k0 >= m) return;
  const Fr ac = DIV ? load_fe<Fr>(a_const, 0) : Fr::zero();
  Fr A = Fr::one(), B = Fr::zero();
  for (size_t k = k0; k < m && k < k0 + chunk; ++k) {
    const Fr a = scan_a<DIV>(arr, ac, k);
    A = Fr::mul(a, A);
    B = Fr::add(Fr::mul(a, B), scan_b<DIV>(arr, m, k));
  }
  store_fe<Fr>(comp, 2 * t, A);
  store_fe<Fr>(comp, 2 * t + 1, B);
}

// one CTA of 256 threads: carry[t] = the x entering chunk t, carry[chunks] = x_m; with check_one, flag = (x_m != 1)
__global__ void __launch_bounds__(256) plonk_scan_carry(const void* comp, size_t chunks, bool start_one, void* carry, bool check_one, unsigned long long* flag) {
  __shared__ Fr runA[256], runB[256], runX[256];
  const uint32_t j = threadIdx.x;
  const size_t per = (chunks + 255) / 256, c0 = j * per < chunks ? j * per : chunks, c1 = c0 + per < chunks ? c0 + per : chunks;
  Fr A = Fr::one(), B = Fr::zero();
  for (size_t c = c0; c < c1; ++c) {
    const Fr a = load_fe<Fr>(comp, 2 * c), b = load_fe<Fr>(comp, 2 * c + 1);
    A = Fr::mul(a, A);
    B = Fr::add(Fr::mul(a, B), b);
  }
  runA[j] = A; runB[j] = B;
  __syncthreads();
  if (j == 0) {
    Fr x = start_one ? Fr::one() : Fr::zero();
    for (int u = 0; u < 256; ++u) { runX[u] = x; x = Fr::add(Fr::mul(runA[u], x), runB[u]); }
    store_fe<Fr>(carry, chunks, x);
    if (check_one && x != Fr::one()) *flag = 1;
  }
  __syncthreads();
  Fr x = runX[j];
  for (size_t c = c0; c < c1; ++c) {
    store_fe<Fr>(carry, c, x);
    x = Fr::add(Fr::mul(load_fe<Fr>(comp, 2 * c), x), load_fe<Fr>(comp, 2 * c + 1));
  }
}

template <bool DIV>
__global__ void __launch_bounds__(256) plonk_scan_apply(void* arr, const void* a_const, size_t m, uint32_t chunk, const void* carry, void* out) {
  const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x, k0 = t * chunk;
  if (k0 >= m) return;
  const Fr ac = DIV ? load_fe<Fr>(a_const, 0) : Fr::zero();
  Fr x = load_fe<Fr>(carry, t);
  for (size_t k = k0; k < m && k < k0 + chunk; ++k) {
    const Fr a = scan_a<DIV>(arr, ac, k), b = scan_b<DIV>(arr, m, k);
    store_fe<Fr>(out, DIV ? m - 1 - k : k, x);
    x = Fr::add(Fr::mul(a, x), b);
  }
}

// ---- round 3: the quotient ----------------------------------------------------------------------------------------------
// On the coset point x_i = 5 w_4n^i (i < 4n), with Z(x w) the value 4 places on:
//   N = a b qm + a ql + b qr + c qo + pi + qc
//     + alpha [(a + beta x + gamma)(b + beta k1 x + gamma)(c + beta k2 x + gamma) z - (a + beta s1 + gamma)(b + beta s2 + gamma)(c + beta s3 + gamma) zw]
//     + alpha^2 (z - 1) L1
//   T = N / Z_H(x), Z_H(x_i) = 5^n w_4^(i mod 4) - 1
// cs: A B C Z PI on the coset (4n apart); kc: Qm Ql Qr Qo Qc S1 S2 S3 L1 on the coset (4n apart)
__global__ void __launch_bounds__(128) plonk_quotient(const void* cs, const void* kc, size_t n4, const void* consts, const void* ch, void* T) {
  const size_t i0 = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) * kQuotChunk;
  if (i0 >= n4) return;
  const Fr beta = ldc(ch, kBeta), gamma = ldc(ch, kGamma), alpha = ldc(ch, kAlpha), a2 = Fr::sqr(alpha);
  const Fr k1 = ldc(consts, kCK1), k2 = ldc(consts, kCK2), w4 = ldc(consts, kCW4);
  Fr x = Fr::mul(ldc(consts, kCGen), pow_u64(w4, i0));
  for (size_t i = i0; i < i0 + kQuotChunk && i < n4; ++i) {
    const Fr a = load_fe_nc<Fr>(cs, i), b = load_fe_nc<Fr>(cs, n4 + i), c = load_fe_nc<Fr>(cs, 2 * n4 + i), z = load_fe_nc<Fr>(cs, 3 * n4 + i);
    const Fr zw = load_fe_nc<Fr>(cs, 3 * n4 + (i + 4) % n4), pi = load_fe_nc<Fr>(cs, 4 * n4 + i);
    Fr q[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) q[k] = load_fe_nc<Fr>(kc, (size_t)k * n4 + i);
    Fr num = Fr::add(Fr::add(Fr::mul(Fr::mul(a, b), q[0]), Fr::mul(a, q[1])), Fr::add(Fr::mul(b, q[2]), Fr::mul(c, q[3])));
    num = Fr::add(num, Fr::add(pi, q[4]));
    const Fr bx = Fr::mul(beta, x);
    const Fr id = Fr::mul(Fr::mul(Fr::mul(Fr::add(Fr::add(a, bx), gamma), Fr::add(Fr::add(b, Fr::mul(bx, k1)), gamma)), Fr::add(Fr::add(c, Fr::mul(bx, k2)), gamma)), z);
    const Fr sg = Fr::mul(Fr::mul(Fr::mul(Fr::add(Fr::add(a, Fr::mul(beta, q[5])), gamma), Fr::add(Fr::add(b, Fr::mul(beta, q[6])), gamma)),
                                  Fr::add(Fr::add(c, Fr::mul(beta, q[7])), gamma)), zw);
    num = Fr::add(num, Fr::mul(alpha, Fr::sub(id, sg)));
    num = Fr::add(num, Fr::mul(a2, Fr::mul(Fr::sub(z, Fr::one()), q[8])));
    store_fe<Fr>(T, i, Fr::mul(num, ldc(consts, kCZhInv + (int)(i & 3))));
    x = Fr::mul(x, w4);
  }
}

// flag = 1 when a coefficient of T at index >= 3n + 6 is nonzero (N was not divisible by Z_H: a gate fails)
__global__ void __launch_bounds__(256) plonk_gate_check(const void* T, size_t from, size_t to, unsigned long long* flag) {
  for (size_t i = from + blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < to; i += (size_t)gridDim.x * blockDim.x)
    if (!load_fe<Fr>(T, i).is_zero()) *flag = 1;
}

// T1 = T[0, n) + b10 X^n, T2 = T[n, 2n) - b10 + b11 X^n, T3 = T[2n, 3n + 6) - b11; each `stride` values apart, zero after
__global__ void __launch_bounds__(256) plonk_split(const void* T, size_t n, size_t stride, const void* blind, void* out) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < stride; i += (size_t)gridDim.x * blockDim.x) {
    Fr t1 = i < n ? load_fe<Fr>(T, i) : (i == n ? blind_at(blind, 10) : Fr::zero());
    Fr t2 = i < n ? load_fe<Fr>(T, n + i) : (i == n ? blind_at(blind, 11) : Fr::zero());
    Fr t3 = i < n + 6 ? load_fe<Fr>(T, 2 * n + i) : Fr::zero();
    if (i == 0) { t2 = Fr::sub(t2, blind_at(blind, 10)); t3 = Fr::sub(t3, blind_at(blind, 11)); }
    store_fe<Fr>(out, i, t1);
    store_fe<Fr>(out, stride + i, t2);
    store_fe<Fr>(out, 2 * stride + i, t3);
  }
}

// ---- round 4: evaluations ------------------------------------------------------------------------------------------------
struct EvalPolys { const void* p[6]; uint32_t len[6]; };  // A B C S1 S2 at xi, Z at xi w
// partial[k * blocks + block] = sum over the block's coefficients of polynomial k = blockIdx.y
__global__ void __launch_bounds__(256) plonk_eval(EvalPolys ps, const void* ch, void* partial) {
  __shared__ Fr red[256];
  const int k = blockIdx.y;
  const Fr x = ldc(ch, k == 5 ? kXiW : kXi);
  const size_t s = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) * kEvalChunk, m = ps.len[k];
  Fr h = Fr::zero();
  if (s < m) {
    for (size_t i = m < s + kEvalChunk ? m : s + kEvalChunk; i-- > s;) h = Fr::add(Fr::mul(h, x), load_fe_nc<Fr>(ps.p[k], i));
    h = Fr::mul(h, pow_u64(x, s));
  }
  red[threadIdx.x] = h;
  __syncthreads();
  for (int o = 128; o; o >>= 1) {
    if ((int)threadIdx.x < o) red[threadIdx.x] = Fr::add(red[threadIdx.x], red[threadIdx.x + o]);
    __syncthreads();
  }
  if (threadIdx.x == 0) store_fe<Fr>(partial, (size_t)k * gridDim.x + blockIdx.x, red[0]);
}

// one CTA of 256: the six evaluations from the partials, xi w, xi^n, Z_H(xi), L1(xi) = Z_H(xi) / (n (xi - 1)) and
// PI(xi) = -(Z_H(xi) / n) sum_i a_i w^i / (xi - w^i) over the public rows
__global__ void __launch_bounds__(256) plonk_eval_finish(const void* partial, uint32_t blocks, const void* a_h, uint32_t n_public, uint32_t log_n,
                                                         const void* consts, void* ch) {
  __shared__ Fr red[256];
  const uint32_t j = threadIdx.x;
  const Fr xi = ldc(ch, kXi), w = ldc(consts, kCW);
  if (j < 6) {
    Fr s = Fr::zero();
    for (uint32_t b = 0; b < blocks; ++b) s = Fr::add(s, load_fe<Fr>(partial, (size_t)j * blocks + b));
    store_fe<Fr>(ch, kEa + j, s);
  }
  Fr acc = Fr::zero();
  for (uint32_t i = j; i < n_public; i += 256) {
    const Fr wi = pow_u64(w, i);
    acc = Fr::add(acc, Fr::mul(Fr::mul(load_fe<Fr>(a_h, i), wi), Fr::inv(Fr::sub(xi, wi))));
  }
  red[j] = acc;
  __syncthreads();
  for (int o = 128; o; o >>= 1) {
    if ((int)j < o) red[j] = Fr::add(red[j], red[j + o]);
    __syncthreads();
  }
  if (j == 0) {
    const Fr xin = pow_u64(xi, 1ull << log_n), zh = Fr::sub(xin, Fr::one()), ninv = ldc(consts, kCNinv);
    store_fe<Fr>(ch, kXin, xin);
    store_fe<Fr>(ch, kZh, zh);
    store_fe<Fr>(ch, kL1, Fr::mul(Fr::mul(zh, ninv), Fr::inv(Fr::sub(xi, Fr::one()))));
    store_fe<Fr>(ch, kPi, Fr::neg(Fr::mul(Fr::mul(zh, ninv), red[0])));
  }
}

// xi w, before the evaluations (the Z evaluation needs it)
__global__ void plonk_xiw(const void* consts, void* ch) {
  if (blockIdx.x || threadIdx.x) return;
  store_fe<Fr>(ch, kXiW, Fr::mul(ldc(ch, kXi), ldc(consts, kCW)));
}

// ---- round 5: the opening numerators -----------------------------------------------------------------------------------
// wx[i] = R_i + v1 A_i + v2 B_i + v3 C_i + v4 S1_i + v5 S2_i (+ the constant kRc0 at i = 0), i < m = n + 6
// wy[i] = Z_i (- eval_zw at i = 0)
// pc: A B C Z coefficients `stride` apart (zero past their length); kq: Qm..S3 coefficients n apart; ts: T1 T2 T3 `stride` apart
__global__ void __launch_bounds__(256) plonk_linearise(const void* pc, const void* kq, const void* ts, size_t n, size_t stride, size_t m, const void* ch, void* wx, void* wy) {
  const Fr rab = ldc(ch, kRab), ea = ldc(ch, kEa), eb = ldc(ch, kEb), ec = ldc(ch, kEc), rz = ldc(ch, kRz), rs3 = ldc(ch, kRs3);
  const Fr zh = ldc(ch, kZh), xin = ldc(ch, kXin), xi2n = Fr::sqr(xin);
  Fr v[5];
  for (int k = 0; k < 5; ++k) v[k] = ldc(ch, kV1 + k);
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < m; i += (size_t)gridDim.x * blockDim.x) {
    const Fr a = load_fe<Fr>(pc, i), b = load_fe<Fr>(pc, stride + i), c = load_fe<Fr>(pc, 2 * stride + i), z = load_fe<Fr>(pc, 3 * stride + i);
    Fr r = Fr::mul(rz, z);
    if (i < n) {
      Fr q[8];
      for (int k = 0; k < 8; ++k) q[k] = load_fe_nc<Fr>(kq, (size_t)k * n + i);
      r = Fr::add(r, Fr::add(Fr::add(Fr::mul(rab, q[0]), Fr::mul(ea, q[1])), Fr::add(Fr::mul(eb, q[2]), Fr::mul(ec, q[3]))));
      r = Fr::add(r, Fr::sub(q[4], Fr::mul(rs3, q[7])));
      r = Fr::add(r, Fr::add(Fr::mul(v[3], q[5]), Fr::mul(v[4], q[6])));
    }
    const Fr t = Fr::add(Fr::add(load_fe<Fr>(ts, i), Fr::mul(xin, load_fe<Fr>(ts, stride + i))), Fr::mul(xi2n, load_fe<Fr>(ts, 2 * stride + i)));
    r = Fr::sub(r, Fr::mul(zh, t));
    r = Fr::add(r, Fr::add(Fr::add(Fr::mul(v[0], a), Fr::mul(v[1], b)), Fr::mul(v[2], c)));
    if (i == 0) r = Fr::add(r, ldc(ch, kRc0));
    store_fe<Fr>(wx, i, r);
    store_fe<Fr>(wy, i, i == 0 ? Fr::sub(z, ldc(ch, kEzw)) : z);
  }
}

unsigned pgrid(b200zk_ctx* ctx, size_t n, unsigned block) {
  size_t g = (n + block - 1) / block, cap = (size_t)ctx->sm_count * 32;
  return (unsigned)(g < cap ? (g ? g : 1) : cap);
}

// ---- host side -------------------------------------------------------------------------------------------------------
int load(b200zk_ctx* ctx, const uint8_t* file, size_t len, int precompute, uint64_t* key) {
  NvtxRange nvtx("b200zk:plonk_zkey_load");
  if (ctx->ntt_root_id != 0)
    return fail(ctx, B200ZK_ERR_INVALID_ARG, "plonk_zkey_load: the context's NTT root is not preset 0 (the snarkjs / ark / gnark root)");
  PlonkLayout L;
  std::string err;
  int rc = plonk_zkey_parse(file, len, &L, &err);
  if (rc) return fail(ctx, rc, err.c_str());
  cudaStream_t st = ctx->stream;
  const size_t n = L.domain_size, n4 = 4 * n, np = n + 6;
  PlonkEntry e;
  e.n_vars = L.n_vars; e.n_public = L.n_public; e.log_n = L.log_n; e.n_additions = L.n_additions; e.n_constraints = L.n_constraints;

  // ---- points: the header's 8 G1 and X_2, PTau; every one on its curve (the coordinates were checked by the parser)
  DevBuf d_hdr;
  B2_CUDA(ctx, cudaMalloc(&d_hdr.p, 8 * 64 + 128));
  B2_CUDA(ctx, cudaMemcpyAsync(d_hdr.p, L.points, 8 * 64 + 128, cudaMemcpyHostToDevice, st));
  BasesEntry pt;
  pt.n = np;
  pt.group = Group::Bn254G1;
  B2_CUDA(ctx, cudaMalloc(&pt.d.p, np * 64 + 32));
  B2_CUDA(ctx, cudaMemcpyAsync(pt.d.p, L.ptau, np * 64, cudaMemcpyHostToDevice, st));
  static const char* kPointName[8] = {"Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3"};
  char msg[160];
  size_t bad = 8;
  rc = b200zk_g1_check_device(ctx, d_hdr.p, 8, st, &bad);
  if (rc == B200ZK_ERR_NOT_ON_CURVE) { snprintf(msg, sizeof msg, "zkey: section 2 (header): %s is not on the curve", kPointName[bad < 8 ? bad : 0]); return fail(ctx, rc, msg); }
  B2_TRY(rc);
  rc = b200zk_g2_check_device(ctx, (const uint8_t*)d_hdr.p + 512, 1, st, &bad);
  if (rc == B200ZK_ERR_NOT_ON_CURVE) return fail(ctx, rc, "zkey: section 2 (header): X_2 is not on the curve");
  B2_TRY(rc);
  rc = b200zk_g1_check_device(ctx, pt.d.p, np, st, &bad);
  if (rc == B200ZK_ERR_NOT_ON_CURVE) { snprintf(msg, sizeof msg, "zkey: section 14 (PTau): point %zu is not on the curve", bad); return fail(ctx, rc, msg); }
  B2_TRY(rc);

  // ---- constants and the verifying key
  B2_CUDA(ctx, cudaMalloc(&e.consts.p, kVkOff + kVkBytes));
  B2_CUDA(ctx, cudaMemcpyAsync(e.consts.p, L.k1, 32, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync((uint8_t*)e.consts.p + 32, L.k2, 32, cudaMemcpyHostToDevice, st));
  Limbs8Arg root;
  B2_TRY(b200zk_ntt_root_preset(0, (uint8_t*)root.v));
  B2_LAUNCH(ctx, plonk_consts, 1, 32, 0, st, root, L.log_n, d_hdr.p, e.consts.p);

  // ---- coefficients (8 x n), S1..S3 on the domain, the 8 and L1 on the coset 5 <w_4n>
  B2_CUDA(ctx, cudaMalloc(&e.coef.p, 8 * n * 32));
  for (int k = 0; k < 8; ++k) {
    const uint8_t* src = k < 5 ? L.q[k] : L.sigma + (size_t)(k - 5) * 5 * n * 32;
    B2_CUDA(ctx, cudaMemcpyAsync((uint8_t*)e.coef.p + (size_t)k * n * 32, src, n * 32, cudaMemcpyHostToDevice, st));
  }
  B2_CUDA(ctx, cudaMalloc(&e.sigma_h.p, 3 * n * 32));
  B2_CUDA(ctx, cudaMemcpyAsync(e.sigma_h.p, (uint8_t*)e.coef.p + 5 * n * 32, 3 * n * 32, cudaMemcpyDeviceToDevice, st));
  for (int k = 0; k < 3; ++k) B2_TRY(ntt_run(ctx, (uint8_t*)e.sigma_h.p + (size_t)k * n * 32, L.log_n, 0, nullptr, st));
  B2_CUDA(ctx, cudaMalloc(&e.coset.p, 9 * n4 * 32));
  B2_CUDA(ctx, cudaMemsetAsync(e.coset.p, 0, 9 * n4 * 32, st));
  for (int k = 0; k < 9; ++k) {
    uint8_t* dst = (uint8_t*)e.coset.p + (size_t)k * n4 * 32;
    if (k < 8) B2_CUDA(ctx, cudaMemcpyAsync(dst, (uint8_t*)e.coef.p + (size_t)k * n * 32, n * 32, cudaMemcpyDeviceToDevice, st));
    else B2_LAUNCH(ctx, plonk_fill, pgrid(ctx, n, 256), 256, 0, st, dst, n, e.consts.p, (int)kCNinv);
    B2_TRY(ntt_run(ctx, dst, L.log_n + 2, B200ZK_NTT_COSET, nullptr, st));
  }

  // ---- maps, and the additions by dependency level (an addition's level is one more than its operands')
  if (L.n_constraints) {
    B2_CUDA(ctx, cudaMalloc(&e.maps.p, 3 * (size_t)L.n_constraints * 4));
    for (int k = 0; k < 3; ++k)
      B2_CUDA(ctx, cudaMemcpyAsync((uint8_t*)e.maps.p + (size_t)k * L.n_constraints * 4, L.map[k], (size_t)L.n_constraints * 4, cudaMemcpyHostToDevice, st));
  }
  const uint32_t na = L.n_additions, n_wtns = L.n_vars - na;
  std::vector<uint8_t> adds;
  if (na) {
    std::vector<uint32_t> level(na), count;
    for (uint32_t i = 0; i < na; ++i) {
      uint32_t s[2];
      memcpy(s, L.additions + kPlonkAddBytes * i, 8);
      uint32_t lv = 0;
      for (uint32_t x : s) if (x >= n_wtns) lv = std::max(lv, level[x - n_wtns] + 1);
      level[i] = lv;
      if (lv >= count.size()) count.resize(lv + 1, 0);
      ++count[lv];
    }
    e.level_off.assign(count.size() + 1, 0);
    for (size_t k = 0; k < count.size(); ++k) e.level_off[k + 1] = e.level_off[k] + count[k];
    std::vector<uint32_t> cursor(e.level_off.begin(), e.level_off.end() - 1);
    adds.assign((size_t)na * (16 + 64), 0);
    uint8_t* f1 = adds.data() + (size_t)na * 16;
    uint8_t* f2 = f1 + (size_t)na * 32;
    for (uint32_t i = 0; i < na; ++i) {
      const uint8_t* a = L.additions + kPlonkAddBytes * i;
      const uint32_t pos = cursor[level[i]]++;
      const uint32_t rec[4] = {n_wtns + i, 0, 0, 0};
      memcpy(adds.data() + 16 * (size_t)pos, rec, 4);
      memcpy(adds.data() + 16 * (size_t)pos + 4, a, 8);
      memcpy(f1 + 32 * (size_t)pos, a + 8, 32);
      memcpy(f2 + 32 * (size_t)pos, a + 40, 32);
    }
    B2_CUDA(ctx, cudaMalloc(&e.adds.p, adds.size()));
    B2_CUDA(ctx, cudaMemcpyAsync(e.adds.p, adds.data(), adds.size(), cudaMemcpyHostToDevice, st));
  }
  e.vk.resize(kVkBytes);
  B2_CUDA(ctx, cudaMemcpyAsync(e.vk.data(), (uint8_t*)e.consts.p + kVkOff, kVkBytes, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));  // adds and vk are host buffers

  // ---- register: PTau (window tables on request), then the key
  B2_TRY(register_bases(ctx, std::move(pt), &e.ptau));
  if (precompute) {
    rc = b200zk_bases_precompute(ctx, e.ptau, 0);
    if (rc) { ctx->bases.erase(e.ptau); return rc; }
  }
  *key = ctx->next_handle++;
  ctx->plonk_keys.emplace(*key, std::move(e));
  return B200ZK_OK;
}

PlonkEntry* find_plonk(b200zk_ctx* ctx, uint64_t key, const char* what) {
  auto it = ctx->plonk_keys.find(key);
  if (it != ctx->plonk_keys.end()) return &it->second;
  fail(ctx, B200ZK_ERR_INVALID_ARG, what);
  return nullptr;
}

// the scan of `m` elements (see the file comment); comp and carry hold 2 and 1 Fr per chunk (+1)
template <bool DIV>
int scan(b200zk_ctx* ctx, void* arr, const void* a_const, size_t m, void* comp, void* carry, unsigned long long* flag, cudaStream_t st) {
  const uint32_t chunk = (uint32_t)std::max<size_t>(32, (m + 65535) / 65536);
  const size_t chunks = (m + chunk - 1) / chunk;
  const unsigned g = (unsigned)((chunks + 255) / 256);
  B2_LAUNCH(ctx, plonk_scan_compose<DIV>, g, 256, 0, st, arr, a_const, m, chunk, comp);
  B2_LAUNCH(ctx, plonk_scan_carry, 1, 256, 0, st, comp, chunks, !DIV, carry, !DIV, flag);
  B2_LAUNCH(ctx, plonk_scan_apply<DIV>, g, 256, 0, st, arr, a_const, m, chunk, carry, arr);
  return B200ZK_OK;
}
size_t scan_chunks(size_t m) { const size_t chunk = std::max<size_t>(32, (m + 65535) / 65536); return (m + chunk - 1) / chunk; }

int prove(b200zk_ctx* ctx, const PlonkEntry& e, const uint8_t* wtns, size_t len, const uint8_t* blinding, cudaStream_t st, uint8_t proof[768]) {
  NvtxRange nvtx("b200zk:plonk_zkey_prove");
  if (ctx->ntt_root_id != 0)
    return fail(ctx, B200ZK_ERR_INVALID_ARG, "plonk_zkey_prove: the context's NTT root is not preset 0 (the snarkjs / ark / gnark root)");
  for (int k = 0; k < 11; ++k) {
    const uint8_t* b = blinding + 32 * k;
    int cmp = 0;
    for (int i = 7; i >= 0 && !cmp; --i) {
      uint32_t v;
      memcpy(&v, b + 4 * i, 4);
      cmp = v < kZkeyR[i] ? -1 : v > kZkeyR[i] ? 1 : 0;
    }
    if (cmp >= 0) {
      char msg[96];
      snprintf(msg, sizeof msg, "plonk_zkey_prove: blinding b%d is >= r", k + 1);
      return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, msg);
    }
  }
  const uint32_t n_wtns = e.n_vars - e.n_additions;
  const uint8_t* values = nullptr;
  std::string err;
  int rc = wtns_parse(wtns, len, n_wtns, &values, &err);
  if (rc) return fail(ctx, rc, err.c_str());
  const BasesEntry* pt = find_bases(ctx, e.ptau, Group::Bn254G1, "plonk_zkey_prove: the key's PTau handle is gone");
  if (!pt) return B200ZK_ERR_INVALID_ARG;

  const size_t n = (size_t)1 << e.log_n, n4 = 4 * n, stride = n + 8;
  // the scans run over n (Z), n + 6 (Wxi) and n + 3 (Wxiw) values; the chunk count is not monotone in m (the chunk
  // grows past 32 values from m > 2^21), so the state is sized for the largest of the three
  const size_t chunks = std::max({scan_chunks(n), scan_chunks(n + 3), scan_chunks(n + 6)}), eval_blocks = (stride + kEvalChunk * 256 - 1) / (kEvalChunk * 256);
  uint8_t *wit, *abc, *pc, *cs, *T, *ts, *zr, *wx, *wy, *comp, *carry, *part, *enc, *ev, *ch, *blind, *tb;
  unsigned long long* status;
  B2_TRY(carve(ctx, ctx->ws_plonk, [&](Carve& c) {
    wit = c.take<uint8_t>(32 * (size_t)e.n_vars); abc = c.take<uint8_t>(3 * 32 * n); pc = c.take<uint8_t>(4 * 32 * stride);
    cs = c.take<uint8_t>(5 * 32 * n4); T = c.take<uint8_t>(32 * n4); ts = c.take<uint8_t>(3 * 32 * stride); zr = c.take<uint8_t>(32 * n);
    wx = c.take<uint8_t>(32 * stride); wy = c.take<uint8_t>(32 * stride); comp = c.take<uint8_t>(64 * chunks); carry = c.take<uint8_t>(32 * (chunks + 1));
    part = c.take<uint8_t>(6 * 32 * eval_blocks + 9 * 128); enc = c.take<uint8_t>(9 * 128 + 6 * 32 + 32); ch = c.take<uint8_t>(32 * kChSlots);
    blind = c.take<uint8_t>(11 * 32); tb = c.take<uint8_t>(512 + 32 * (size_t)e.n_public + 192); status = c.take<unsigned long long>(4);
  }));
  uint8_t* msm_part = part + 6 * 32 * eval_blocks;  // 9 XYZZ partials, 128 bytes each
  ev = enc + 9 * 128;
  auto commit = [&](int slot, const void* scalars, size_t count) -> int {
    B2_TRY(msm_run_g1(ctx, pt->d.p, scalars, count, B200ZK_SCALARS_MONT, st, msm_part + 128 * slot, pt->table_c, pt->n));
    return msm_encode_g1(ctx, msm_part + 128 * slot, 1, 0, st, enc + 128 * slot);
  };
  const uint8_t* consts = (const uint8_t*)e.consts.p;
  uint8_t* pcA = pc; uint8_t* pcZ = pc + 3 * 32 * stride;
  uint8_t* csPI = cs + 4 * 32 * n4;
  // with profiling, events at the round boundaries (b200zk_plonk_last_round_ms)
  auto mark = [&](int k) -> int { if (ctx->profiling && ctx->ev_plonk[k]) B2_CUDA(ctx, cudaEventRecord(ctx->ev_plonk[k], st)); return B200ZK_OK; };

  // ---- round 1: the witness, the additions, a b c, their blinded coefficients and commitments
  B2_TRY(mark(0));
  B2_CUDA(ctx, cudaMemcpyAsync(wit, values, 32 * (size_t)n_wtns, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(blind, blinding, 11 * 32, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(status, 0, 32, st));
  B2_CUDA(ctx, cudaMemsetAsync(status, 0xff, 8, st));
  B2_LAUNCH(ctx, plonk_range_check, pgrid(ctx, n_wtns, 256), 256, 0, st, wit, (size_t)n_wtns, status);
  if (e.n_additions) {
    const uint4* rec = (const uint4*)e.adds.p;
    const uint8_t* f1 = (const uint8_t*)e.adds.p + 16 * (size_t)e.n_additions;
    const uint8_t* f2 = f1 + 32 * (size_t)e.n_additions;
    for (size_t k = 0; k + 1 < e.level_off.size(); ++k) {
      const uint32_t b = e.level_off[k], en = e.level_off[k + 1];
      B2_LAUNCH(ctx, plonk_additions, (en - b + 255) / 256, 256, 0, st, rec, f1, f2, b, en, wit);
    }
  }
  B2_CUDA(ctx, cudaMemsetAsync(pc, 0, 4 * 32 * stride, st));
  B2_CUDA(ctx, cudaMemsetAsync(cs, 0, 5 * 32 * n4, st));
  B2_LAUNCH(ctx, plonk_gather, pgrid(ctx, n, 256), 256, 0, st, (const uint32_t*)e.maps.p, e.n_constraints, e.n_public, n, wit, abc, e.n_public ? csPI : nullptr);
  static const int kBlindIdx[4][3] = {{2, 1, 0}, {4, 3, 0}, {6, 5, 0}, {9, 8, 7}};
  for (int k = 0; k < 3; ++k) {
    uint8_t* p = pc + (size_t)k * 32 * stride;
    B2_CUDA(ctx, cudaMemcpyAsync(p, abc + (size_t)k * 32 * n, 32 * n, cudaMemcpyDeviceToDevice, st));
    B2_TRY(ntt_run(ctx, p, e.log_n, B200ZK_NTT_INVERSE, nullptr, st));
    B2_LAUNCH(ctx, plonk_blind, 1, 32, 0, st, p, n, blind, 2, kBlindIdx[k][0], kBlindIdx[k][1], 0);
    B2_TRY(commit(k, p, n + 2));
  }
  B2_LAUNCH(ctx, plonk_transcript, 1, 32, 0, st, 0, consts, abc, e.n_public, enc, ch, tb, ev);

  // ---- round 2: Z
  B2_TRY(mark(1));
  B2_LAUNCH(ctx, plonk_perm_ratio, (unsigned)(((n + kRatioChunk - 1) / kRatioChunk + 127) / 128), 128, 0, st, abc, e.sigma_h.p, n, consts, ch, zr);
  B2_TRY(scan<false>(ctx, zr, nullptr, n, comp, carry, status + 1, st));
  B2_CUDA(ctx, cudaMemcpyAsync(pcZ, zr, 32 * n, cudaMemcpyDeviceToDevice, st));
  B2_TRY(ntt_run(ctx, pcZ, e.log_n, B200ZK_NTT_INVERSE, nullptr, st));
  B2_LAUNCH(ctx, plonk_blind, 1, 32, 0, st, pcZ, n, blind, 3, kBlindIdx[3][0], kBlindIdx[3][1], kBlindIdx[3][2]);
  B2_TRY(commit(3, pcZ, n + 3));
  B2_LAUNCH(ctx, plonk_transcript, 1, 32, 0, st, 1, consts, abc, e.n_public, enc, ch, tb, ev);

  // ---- round 3: T on the coset, its coefficients, the gate check, T1 T2 T3
  B2_TRY(mark(2));
  for (int k = 0; k < 4; ++k) {
    uint8_t* dst = cs + (size_t)k * 32 * n4;
    B2_CUDA(ctx, cudaMemcpyAsync(dst, pc + (size_t)k * 32 * stride, 32 * stride, cudaMemcpyDeviceToDevice, st));
    B2_TRY(ntt_run(ctx, dst, e.log_n + 2, B200ZK_NTT_COSET, nullptr, st));
  }
  if (e.n_public) {
    B2_TRY(ntt_run(ctx, csPI, e.log_n, B200ZK_NTT_INVERSE, nullptr, st));
    B2_TRY(ntt_run(ctx, csPI, e.log_n + 2, B200ZK_NTT_COSET, nullptr, st));
  }
  B2_LAUNCH(ctx, plonk_quotient, (unsigned)(((n4 + kQuotChunk - 1) / kQuotChunk + 127) / 128), 128, 0, st, cs, e.coset.p, n4, consts, ch, T);
  B2_TRY(ntt_run(ctx, T, e.log_n + 2, B200ZK_NTT_INVERSE | B200ZK_NTT_COSET, nullptr, st));
  B2_LAUNCH(ctx, plonk_gate_check, pgrid(ctx, n - 6, 256), 256, 0, st, T, 3 * n + 6, n4, status + 2);
  B2_LAUNCH(ctx, plonk_split, pgrid(ctx, stride, 256), 256, 0, st, T, n, stride, blind, ts);
  B2_TRY(commit(4, ts, n + 1));
  B2_TRY(commit(5, ts + 32 * stride, n + 1));
  B2_TRY(commit(6, ts + 64 * stride, n + 6));
  B2_LAUNCH(ctx, plonk_transcript, 1, 32, 0, st, 2, consts, abc, e.n_public, enc, ch, tb, ev);

  // ---- round 4: the evaluations
  B2_TRY(mark(3));
  B2_LAUNCH(ctx, plonk_xiw, 1, 32, 0, st, consts, ch);
  EvalPolys ps;
  const uint8_t* kq = (const uint8_t*)e.coef.p;
  const void* polys[6] = {pcA, pcA + 32 * stride, pcA + 64 * stride, kq + 5 * 32 * n, kq + 6 * 32 * n, pcZ};
  const uint32_t lens[6] = {(uint32_t)n + 2, (uint32_t)n + 2, (uint32_t)n + 2, (uint32_t)n, (uint32_t)n, (uint32_t)n + 3};
  for (int k = 0; k < 6; ++k) { ps.p[k] = polys[k]; ps.len[k] = lens[k]; }
  B2_LAUNCH(ctx, plonk_eval, dim3((unsigned)eval_blocks, 6), 256, 0, st, ps, ch, part);
  B2_LAUNCH(ctx, plonk_eval_finish, 1, 256, 0, st, part, (uint32_t)eval_blocks, abc, e.n_public, e.log_n, consts, ch);
  B2_LAUNCH(ctx, plonk_transcript, 1, 32, 0, st, 3, consts, abc, e.n_public, enc, ch, tb, ev);

  // ---- round 5: Wxi and Wxiw
  B2_TRY(mark(4));
  B2_LAUNCH(ctx, plonk_linearise, pgrid(ctx, n + 6, 256), 256, 0, st, pc, kq, ts, n, stride, n + 6, ch, wx, wy);
  B2_TRY(scan<true>(ctx, wx, ch + 32 * kXi, n + 6, comp, carry, nullptr, st));
  B2_TRY(scan<true>(ctx, wy, ch + 32 * kXiW, n + 3, comp, carry, nullptr, st));
  B2_TRY(commit(7, wx, n + 5));
  B2_TRY(commit(8, wy, n + 2));

  B2_TRY(mark(5));
  // ---- the proof and the three checks in one copy
  uint8_t* h = ctx->h_pinned;
  B2_CUDA(ctx, cudaMemcpy2DAsync(h, 64, enc, 128, 64, 9, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(h + 576, ev, 192, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(h + 768, status, 24, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (ctx->profiling && ctx->ev_plonk[5])
    for (int k = 0; k < 5; ++k) B2_CUDA(ctx, cudaEventElapsedTime(&ctx->plonk_round_ms[k], ctx->ev_plonk[k], ctx->ev_plonk[k + 1]));
  unsigned long long flags[3];
  memcpy(flags, h + 768, 24);
  if (flags[0] != ~0ull) {
    char msg[128];
    snprintf(msg, sizeof msg, "wtns: section 2: value %llu is >= r", flags[0]);
    return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, msg);
  }
  if (flags[1]) return fail(ctx, B200ZK_ERR_INVALID_ARG, "plonk_zkey_prove: witness does not satisfy the copy constraints");
  if (flags[2]) return fail(ctx, B200ZK_ERR_INVALID_ARG, "plonk_zkey_prove: witness does not satisfy the gates");
  memcpy(proof, h, 768);
  return B200ZK_OK;
}

}  // namespace
}  // namespace b200zk

using namespace b200zk;

extern "C" {

int b200zk_plonk_zkey_load(b200zk_ctx* ctx, const void* zkey, size_t len, int precompute, uint64_t* key) {
  if (!ctx || !key) return fail(ctx, B200ZK_ERR_INVALID_ARG, "plonk_zkey_load: null argument");
  DeviceGuard guard(ctx);
  return load(ctx, (const uint8_t*)zkey, len, precompute, key);
}

int b200zk_plonk_zkey_free(b200zk_ctx* ctx, uint64_t key) {
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  DeviceGuard guard(ctx);
  PlonkEntry* e = find_plonk(ctx, key, "plonk_zkey_free: unknown key");
  if (!e) return B200ZK_ERR_INVALID_ARG;
  B2_CUDA(ctx, cudaDeviceSynchronize());
  ctx->bases.erase(e->ptau);
  ctx->plonk_keys.erase(key);
  return B200ZK_OK;
}

int b200zk_plonk_zkey_info(b200zk_ctx* ctx, uint64_t key, uint32_t* n_vars, uint32_t* n_public, uint32_t* log_n, uint8_t* vk, size_t vk_len) {
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  const PlonkEntry* e = find_plonk(ctx, key, "plonk_zkey_info: unknown key");
  if (!e) return B200ZK_ERR_INVALID_ARG;
  if (n_vars) *n_vars = e->n_vars;
  if (n_public) *n_public = e->n_public;
  if (log_n) *log_n = e->log_n;
  if (vk) {
    if (vk_len < kVkBytes) return fail(ctx, B200ZK_ERR_INVALID_ARG, "plonk_zkey_info: vk buffer shorter than 736 bytes");
    memcpy(vk, e->vk.data(), kVkBytes);
  }
  return B200ZK_OK;
}

int b200zk_plonk_zkey_prove(b200zk_ctx* ctx, uint64_t key, const void* wtns, size_t len, const uint8_t blinding[11 * 32], void* stream, uint8_t proof[768]) {
  if (!ctx || !blinding || !proof) return fail(ctx, B200ZK_ERR_INVALID_ARG, "plonk_zkey_prove: null argument");
  DeviceGuard guard(ctx);
  const PlonkEntry* e = find_plonk(ctx, key, "plonk_zkey_prove: unknown key");
  if (!e) return B200ZK_ERR_INVALID_ARG;
  return prove(ctx, *e, (const uint8_t*)wtns, len, blinding, pick_stream(ctx, stream), proof);
}

int b200zk_plonk_last_round_ms(b200zk_ctx* ctx, float out_ms[5]) {
  if (!ctx || !out_ms) return fail(ctx, B200ZK_ERR_INVALID_ARG, "plonk_last_round_ms: null argument");
  if (!ctx->profiling) return fail(ctx, B200ZK_ERR_INVALID_ARG, "plonk_last_round_ms: profiling is off");
  memcpy(out_ms, ctx->plonk_round_ms, sizeof ctx->plonk_round_ms);
  return B200ZK_OK;
}

}  // extern "C"
