// kzg_cells.cu -- EIP-7594 (PeerDAS) cells on the device: the cell extension of a blob (c-kzg compute_cells) and the
// scalars of the batched cell-proof check (verify_cell_kzg_proof_batch, whose pairing lives in bls_pairing.cu):
//   crates/common/crypto/kzg.rs:72-113          verify_cell_kzg_proof_batch, compute_cells
//   crates/common/types/blobs_bundle.rs:152-173 BlobsBundle::verify_kzg_proofs, wrapper version 1
// A blob lists p's values on the 4096 roots of unity in bit-reversed order.  Its extension lists p on the 8192nd roots in
// bit-reversed order: brp13(i) = 2 brp12(i) for i < 4096, so the first half is the blob itself, and brp13(4096 + j) =
// 2 brp12(j) + 1, so the second half is p on the coset w_8192 <w_4096>, again in bit-reversed order.  That half is one
// size-4096 NTT of the coefficients c_i w_8192^i: the zero-padded size-8192 NTT of the spec splits into that and the blob.
// So each blob takes an inverse and a forward NTT of size 4096 (128 KiB of Fr381, one CTA's shared memory), and the
// 256 KiB of the full extension never has to sit in one CTA.
#include "bls12.cuh"
#include <algorithm>
#include <cstring>
#include <vector>

namespace b200zk {
namespace {

constexpr uint32_t kN = 4096;       // FIELD_ELEMENTS_PER_BLOB
constexpr uint32_t kExtN = 8192;    // FIELD_ELEMENTS_PER_EXT_BLOB
constexpr uint32_t kCellN = 64;     // FIELD_ELEMENTS_PER_CELL
constexpr uint32_t kCells = 128;    // CELLS_PER_EXT_BLOB
constexpr uint32_t kThreads = 256;  // one CTA per blob: 8 butterflies per thread and stage
constexpr size_t kSmem = kN * 32;   // the blob's 4096 elements

B2_D Fr381 tw_at(const void* tw, uint32_t i) { return load_fe_nc<Fr381>(tw, i); }
B2_D uint32_t brp7(uint32_t c) { return __brev(c) >> 25; }

// tw[i] = w^i for i < 8192, w = 7^((r-1)/8192); tw[8192] = 1/4096 = r - (r-1)/4096.  Montgomery form.  One thread per
// entry, each deriving w from its definition: a one-off per context.  w^2 is the blob domain's root (kzg_roots_build).
__global__ void __launch_bounds__(256) kzg_cells_tw_build(void* __restrict__ tw) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > kExtN) return;
  const uint32_t sh = i == kExtN ? 12 : 13;  // (r - 1) >> sh (r - 1 = r with limb 0 cleared)
  Fr381 e;
#pragma unroll
  for (int k = 0; k < 8; ++k) e.v[k] = ((k ? bls_r_limb(k) : 0u) >> sh) | (k < 7 ? bls_r_limb(k + 1) << (32 - sh) : 0u);
  if (i == kExtN) { store_fe(tw, i, Fr381::to_mont(Fr381::sub(Fr381::zero(), e))); return; }
  Fr381 c = Fr381::zero();
  c.v[0] = 7;
  Fr381 base = Fr381::pow(Fr381::to_mont(c), e.v), acc = Fr381::one();
#pragma unroll 1
  for (uint32_t x = i; x; x >>= 1) {
    if (x & 1) acc = Fr381::mul(acc, base);
    base = Fr381::sqr(base);
  }
  store_fe(tw, i, acc);
}

// In place over the 4096 elements in s, all threads of the CTA, s written and synchronised by the caller.  Twiddles of a
// butterfly span 2h are powers of w_2h = w_8192^(8192 / 2h).  Elements may be canonical or Montgomery: the twiddles are
// Montgomery, so mul keeps the input's form.
// Inverse, Cooley-Tukey: bit-reversed values in, natural-order coefficients out, times 4096 (no scaling).  With size < 4096
// only the first log2(size) stages run: independent inverse NTTs of that size (times size) on each block of size elements.
B2_D void ntt_inverse_brp(uint4* s, const void* tw, uint32_t size = kN) {
  for (uint32_t h = 1; h < size; h <<= 1) {
    const uint32_t step = kExtN / (2 * h);
#pragma unroll 1
    for (uint32_t b = threadIdx.x; b < kN / 2; b += kThreads) {
      const uint32_t j = b & (h - 1), i0 = 2 * b - j, i1 = i0 + h;
      const Fr381 u = load_fe<Fr381>(s, i0), v = Fr381::mul(load_fe<Fr381>(s, i1), tw_at(tw, (kExtN - j * step) & (kExtN - 1)));
      store_fe(s, i0, Fr381::add(u, v));
      store_fe(s, i1, Fr381::sub(u, v));
    }
    __syncthreads();
  }
}
// Forward, Gentleman-Sande: natural-order coefficients in, values on the 4096 roots out in bit-reversed order
B2_D void ntt_forward_brp(uint4* s, const void* tw) {
  for (uint32_t h = kN / 2; h >= 1; h >>= 1) {
    const uint32_t step = kExtN / (2 * h);
#pragma unroll 1
    for (uint32_t b = threadIdx.x; b < kN / 2; b += kThreads) {
      const uint32_t j = b & (h - 1), i0 = 2 * b - j, i1 = i0 + h;
      const Fr381 u = load_fe<Fr381>(s, i0), v = load_fe<Fr381>(s, i1);
      store_fe(s, i0, Fr381::add(u, v));
      store_fe(s, i1, Fr381::mul(Fr381::sub(u, v), tw_at(tw, j * step)));
    }
    __syncthreads();
  }
}

// blob (4096 x 32-byte big-endian, checked < r) -> s as canonical limbs
B2_D void load_blob(uint4* s, const uint8_t* blob) {
  for (uint32_t i = threadIdx.x; i < kN; i += kThreads) store_fe(s, i, load_be32(blob + 32 * i));
  __syncthreads();
}

// One CTA per blob: its 128 cells (8192 x 32-byte big-endian).  Cells 0..63 are the blob's bytes; cells 64..127 are
// the forward NTT of c_i w_8192^i / 4096.  Values stay canonical throughout.
__global__ void __launch_bounds__(kThreads, 1) kzg_cells_extend(const uint8_t* __restrict__ blobs, const void* __restrict__ tw, uint8_t* __restrict__ cells) {
  extern __shared__ uint4 cells_smem[];
  const uint8_t* blob = blobs + (size_t)blockIdx.x * kN * 32;
  uint8_t* out = cells + (size_t)blockIdx.x * kExtN * 32;
  for (uint32_t i = threadIdx.x; i < 2 * kN; i += kThreads)
    reinterpret_cast<uint4*>(out)[i] = __ldg(reinterpret_cast<const uint4*>(blob) + i);
  load_blob(cells_smem, blob);
  ntt_inverse_brp(cells_smem, tw);
  const Fr381 ninv = tw_at(tw, kExtN);
  for (uint32_t i = threadIdx.x; i < kN; i += kThreads)
    store_fe(cells_smem, i, Fr381::mul(Fr381::mul(load_fe<Fr381>(cells_smem, i), tw_at(tw, i)), ninv));
  __syncthreads();
  ntt_forward_brp(cells_smem, tw);
  for (uint32_t i = threadIdx.x; i < kN; i += kThreads) store_be32(out + 32 * (kN + i), load_fe<Fr381>(cells_smem, i));
}

// ---- the batched cell-proof check --------------------------------------------------------------------------------------
// Cell k (global index 128 b + c over blob b, cell c) covers the coset h_c <w_64>, h_c = w_8192^brp7(c), the roots of
// X^64 - s_c with s_c = h_c^64 = w_8192^(64 brp7(c)).  Its interpolation polynomial is I_k = p_b mod (X^64 - s_c):
// coefficient j is sum_m c_b[64 m + j] s_c^m.  With the challenge r,
//   A = sum_k r^k I_k,  A_j = sum_b r^(128 b) sum_m c_b[64 m + j] V_m,  V_m = sum_c r^c s_c^m,
// so one 64 x 64 product per blob gives its share of A, and A of degree < 64 evaluated on the 4096 bit-reversed roots
// is the scalar vector of [A(tau)]1 over the Lagrange setup.

// weights = V_0 .. V_63 (V_0 = sum_c r^c), then r; Montgomery.  One CTA of 65 threads.
__global__ void __launch_bounds__(96) kzg_cells_weights(const uint8_t* __restrict__ r_be, const void* __restrict__ tw, void* __restrict__ weights) {
  const uint32_t m = threadIdx.x;
  if (m > kCellN) return;
  const Fr381 r = Fr381::to_mont(load_be32(r_be));
  if (m == kCellN) { store_fe(weights, m, r); return; }
  Fr381 acc = Fr381::zero(), rc = Fr381::one();
#pragma unroll 1
  for (uint32_t c = 0; c < kCells; ++c) {
    acc = Fr381::add(acc, Fr381::mul(rc, tw_at(tw, (kCellN * brp7(c) * m) & (kExtN - 1))));
    rc = Fr381::mul(rc, r);
  }
  store_fe(weights, m, acc);
}

// One CTA per blob: partial[64 b + j] = r^(128 b) / 4096 sum_m c'_b[64 m + j] V_m (canonical), c' = 4096 c the unscaled
// inverse NTT
__global__ void __launch_bounds__(kThreads, 1) kzg_cells_interp(const uint8_t* __restrict__ blobs, const void* __restrict__ tw, const void* __restrict__ weights,
                                                               void* __restrict__ partial) {
  extern __shared__ uint4 cells_smem[];
  __shared__ uint4 s_scale[2];
  if (threadIdx.x == 0) {
    const uint32_t e[8] = {kCells * blockIdx.x, 0, 0, 0, 0, 0, 0, 0};
    store_fe(s_scale, 0, Fr381::mul(Fr381::pow(load_fe_nc<Fr381>(weights, kCellN), e), tw_at(tw, kExtN)));
  }
  load_blob(cells_smem, blobs + (size_t)blockIdx.x * kN * 32);
  ntt_inverse_brp(cells_smem, tw);
  const uint32_t j = threadIdx.x;
  if (j >= kCellN) return;
  Fr381 acc = Fr381::zero();
#pragma unroll 1
  for (uint32_t m = 0; m < kN / kCellN; ++m) acc = Fr381::add(acc, Fr381::mul(load_fe<Fr381>(cells_smem, kCellN * m + j), load_fe_nc<Fr381>(weights, m)));
  store_fe(partial, (size_t)kCellN * blockIdx.x + j, Fr381::mul(acc, load_fe<Fr381>(s_scale, 0)));
}

// One CTA: A_j = sum_b partial[64 b + j], zero-padded to 4096 and evaluated on the bit-reversed roots; out: canonical
// little-endian limbs, the scalars of the Lagrange-setup MSM
__global__ void __launch_bounds__(kThreads, 1) kzg_cells_interp_eval(const void* __restrict__ partial, size_t n, const void* __restrict__ tw, void* __restrict__ s_setup) {
  extern __shared__ uint4 cells_smem[];
  for (uint32_t i = threadIdx.x; i < kN; i += kThreads) {
    Fr381 a = Fr381::zero();
    if (i < kCellN)
      for (size_t b = 0; b < n; ++b) a = Fr381::add(a, load_fe<Fr381>(partial, kCellN * b + i));
    store_fe(cells_smem, i, a);
  }
  __syncthreads();
  ntt_forward_brp(cells_smem, tw);
  for (uint32_t i = threadIdx.x; i < kN; i += kThreads) store_fe(s_setup, i, load_fe<Fr381>(cells_smem, i));
}

// k < n: s_lin[k] = r^(128 k) V_0, commitment k's scalar; n <= k < 129 n, cell q = k - n: s_lin[k] = r^q s_(q mod 128)
// and s_proof[q] = r^q.  Canonical little-endian limbs.
__global__ void __launch_bounds__(256) kzg_cells_scalars(const void* __restrict__ tw, const void* __restrict__ weights, size_t n,
                                                         void* __restrict__ s_proof, void* __restrict__ s_lin) {
  const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (k >= (kCells + 1) * n) return;
  const size_t q = k < n ? kCells * k : k - n;
  const uint32_t e[8] = {(uint32_t)q, (uint32_t)((uint64_t)q >> 32), 0, 0, 0, 0, 0, 0};
  const Fr381 rq = Fr381::pow(load_fe_nc<Fr381>(weights, kCellN), e);
  if (k < n) { store_fe(s_lin, k, Fr381::from_mont(Fr381::mul(rq, load_fe_nc<Fr381>(weights, 0)))); return; }
  store_fe(s_proof, q, Fr381::from_mont(rq));
  store_fe(s_lin, k, Fr381::from_mont(Fr381::mul(rq, tw_at(tw, kCellN * brp7((uint32_t)(q % kCells))))));
}

// ---- the same check over arbitrary cells (b200zk_kzg_verify_cells) ---------------------------------------------------
// Cell k carries its own commitment (index i_k among the deduplicated ones) and cell index c_k.  The interpolant of a
// cell on its coset h_c <w_64> comes from its values alone: its values at h_c w_64^brp6(t) are y[t], so the inverse NTT
// of size 64 (bit-reversed in, natural out) gives g(Y) = I(h_c Y), and I's coefficient j is g_j h_c^-j / 64.  Cells that
// share a cell index share the coset, so A = sum_k r^k I_k is one such interpolation per cell index c that occurs, of
// agg_c = sum_(k: c_k = c) r^k y_k, and its coefficients go through kzg_cells_interp_eval like the per-blob shares above.

// one thread per cell: rpow[k] = r^k (Montgomery); s_proof[k] = r^k and s_lin[n_commit + k] = r^k h_(c_k)^64 (canonical)
__global__ void __launch_bounds__(256) kzg_vcells_powers(const uint8_t* __restrict__ r_be, const void* __restrict__ tw, const uint32_t* __restrict__ idx,
                                                          size_t n, size_t n_commit, void* __restrict__ rpow, void* __restrict__ s_proof, void* __restrict__ s_lin) {
  const size_t k = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (k >= n) return;
  const uint32_t e[8] = {(uint32_t)k, (uint32_t)((uint64_t)k >> 32), 0, 0, 0, 0, 0, 0};
  const Fr381 rk = Fr381::pow(Fr381::to_mont(load_be32(r_be)), e);
  store_fe(rpow, k, rk);
  store_fe(s_proof, k, Fr381::from_mont(rk));
  store_fe(s_lin, n_commit + k, Fr381::from_mont(Fr381::mul(rk, tw_at(tw, kCellN * brp7(idx[k])))));
}

// one thread per deduplicated commitment i: s_lin[i] = sum r^k over its cells (by_commit[off[i] .. off[i + 1]))
__global__ void __launch_bounds__(256) kzg_vcells_weights(const uint32_t* __restrict__ off, const uint32_t* __restrict__ by_commit, size_t n_commit,
                                                           const void* __restrict__ s_proof, void* __restrict__ s_lin) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n_commit) return;
  Fr381 w = Fr381::zero();
#pragma unroll 1
  for (uint32_t q = off[i]; q < off[i + 1]; ++q) w = Fr381::add(w, load_fe_nc<Fr381>(s_proof, by_commit[q]));
  store_fe(s_lin, i, w);
}

// One CTA per 64 of the cell indices that occur (columns[q], q < n_cols; cells by_column[off[q] .. off[q + 1])):
// partial[64 q + j] = coefficient j of the interpolant of agg_q on its coset (canonical), the layout of kzg_cells_interp
__global__ void __launch_bounds__(kThreads, 1) kzg_vcells_columns(const uint8_t* __restrict__ cells, const void* __restrict__ rpow,
                                                                 const uint32_t* __restrict__ off, const uint32_t* __restrict__ by_column,
                                                                 const uint32_t* __restrict__ columns, size_t n_cols, const void* __restrict__ tw,
                                                                 void* __restrict__ partial) {
  extern __shared__ uint4 cells_smem[];
  const size_t first = (size_t)kCellN * blockIdx.x;
  for (uint32_t e = threadIdx.x; e < kN; e += kThreads) {
    const size_t q = first + e / kCellN;
    Fr381 acc = Fr381::zero();
    if (q < n_cols) {
#pragma unroll 1
      for (uint32_t s = off[q]; s < off[q + 1]; ++s) {
        const uint32_t k = by_column[s];
        acc = Fr381::add(acc, Fr381::mul(load_be32(cells + kCellN * 32 * (size_t)k + 32 * (e % kCellN)), load_fe_nc<Fr381>(rpow, k)));
      }
    }
    store_fe(cells_smem, e, acc);
  }
  __syncthreads();
  ntt_inverse_brp(cells_smem, tw, kCellN);
  Fr381 inv64 = tw_at(tw, kExtN);  // 1/4096, doubled six times
#pragma unroll 1
  for (int k = 0; k < 6; ++k) inv64 = Fr381::dbl(inv64);
  for (uint32_t e = threadIdx.x; e < kN; e += kThreads) {
    const size_t q = first + e / kCellN;
    if (q >= n_cols) break;
    const uint32_t j = e % kCellN;
    const Fr381 unshift = Fr381::mul(tw_at(tw, (kExtN - brp7(columns[q]) * j) & (kExtN - 1)), inv64);
    store_fe(partial, first * kCellN + e, Fr381::mul(load_fe<Fr381>(cells_smem, e), unshift));
  }
}

// ---- cell proofs by FK20 (c-kzg compute_cells_and_kzg_proofs) --------------------------------------------------------
// pi_k = [q_k(tau)]1, q_k = (p - I_k) / (X^64 - s_k), is sum_(m=1..63) s_k^(m-1) T_m with the Toeplitz sums
//   T_m = sum_(i <= 4095 - 64 m) c_(i + 64 m) [tau^i]1 = sum_b sum_(a <= 63 - m) C_b[a + m] S_b[a],
// C_b[t] = c_(64 t + b), S_b[a] = [tau^(64 a + b)]1.  Per column b that is a circular convolution of length 128 of C_b
// (zero-padded) with S''_b (S''_b[0] = S_b[0], S''_b[128 - a] = S_b[a] for a = 1..63, else O) that never wraps for m < 64, so
//   table[b] = DFT(S''_b) (once per setup),  u = sum_b DFT(C_b) table[b],  T_m = DFT^-1(u)[m],
// and the 128 proofs are one more DFT of (T_1 .. T_63, O ..), since s_k = w_128^brp7(k).  All DFTs have size 128 and root
// w_128 = w_8192^64.  Forward DFTs are Gentleman-Sande (natural in, bit-reversed out) and the inverse is Cooley-Tukey
// (bit-reversed in, natural out), as the NTTs above: the column DFTs and the table are both bit-reversed, the pointwise
// sums need no permutation, and the last DFT leaves pi_k at position k.  tests/fk20_ref.py restates every step in scalars.
constexpr uint32_t kDft = 128;            // the circulant's size
constexpr uint32_t kColGroup = 16;        // columns per pass of kzg_fk20_columns: 4096 coefficients + 16 x 128 in shared memory
constexpr size_t kColSmem = (kN + kColGroup * kDft) * 32;
constexpr uint32_t kMsmWarps = 4;         // kzg_fk20_msm: one warp per (blob, position) MSM of 64 terms

B2_D XYZZ<Fp381> xyzz_neg(const XYZZ<Fp381>& p) { return {p.x, Fp381::neg(p.y), p.zz, p.zzz}; }

// k P for a canonical scalar k < r < 2^255 (double-and-add, MSB first): the twiddle products of the G1 DFTs
B2_D XYZZ<Fp381> xyzz_mul_fr(const XYZZ<Fp381>& p, const Fr381& k) {
  XYZZ<Fp381> acc = XYZZ<Fp381>::identity();
#pragma unroll 1
  for (int i = 254; i >= 0; --i) {
    acc = xyzz_dbl(acc);
    if ((k.v[i >> 5] >> (i & 31)) & 1) xyzz_add(acc, p);
  }
  return acc;
}

// In place over 128 XYZZ points in s, 64 threads (one butterfly each per stage), s written and synchronised by the caller.
// Forward, Gentleman-Sande: natural order in, DFT[brp7(i)] at position i.  A butterfly of twiddle 1 (j = 0) multiplies nothing.
B2_D void g1_dft_forward(void* s, const void* tw) {
  for (uint32_t h = kDft / 2; h >= 1; h >>= 1) {
    const uint32_t b = threadIdx.x, j = b & (h - 1), i0 = 2 * b - j, i1 = i0 + h;
    XYZZ<Fp381> u = load_xyzz<Fp381>(s, i0);
    const XYZZ<Fp381> v = load_xyzz<Fp381>(s, i1);
    XYZZ<Fp381> d = xyzz_neg(v);
    xyzz_add(d, u);
    xyzz_add(u, v);
    store_xyzz<Fp381>(s, i0, u);
    if (j) d = xyzz_mul_fr(d, Fr381::from_mont(tw_at(tw, j * (kExtN / (2 * h)))));
    store_xyzz<Fp381>(s, i1, d);
    __syncthreads();
  }
}
// Inverse, Cooley-Tukey, root w_128^-1, unscaled: bit-reversed order in, natural order out
B2_D void g1_dft_inverse(void* s, const void* tw) {
  for (uint32_t h = 1; h < kDft; h <<= 1) {
    const uint32_t b = threadIdx.x, j = b & (h - 1), i0 = 2 * b - j, i1 = i0 + h;
    XYZZ<Fp381> v = load_xyzz<Fp381>(s, i1);
    if (j) v = xyzz_mul_fr(v, Fr381::from_mont(tw_at(tw, kExtN - j * (kExtN / (2 * h)))));
    XYZZ<Fp381> u = load_xyzz<Fp381>(s, i0), d = xyzz_neg(v);
    xyzz_add(d, u);
    xyzz_add(u, v);
    store_xyzz<Fp381>(s, i0, u);
    store_xyzz<Fp381>(s, i1, d);
    __syncthreads();
  }
}

// One CTA of 64 threads per column b: table[128 b + i] = DFT(S''_b)[brp7(i)] as native affine points.  mono: the monomial
// setup's points [tau^i]1 (native affine, the first 4096 entries of the handle whether or not it holds window tables).
__global__ void __launch_bounds__(kDft / 2, 1) kzg_fk20_table(const void* __restrict__ mono, const void* __restrict__ tw, void* __restrict__ table) {
  __shared__ uint4 s_pts[kDft * 12];  // 128 XYZZ points, 192 bytes each
  const uint32_t b = blockIdx.x, t = threadIdx.x;
  // k = t: S''[0] = S_b[0], then O; k = 64 + t: O at 64, then S_b[a] for a = 128 - k = 64 - t
  store_xyzz<Fp381>(s_pts, t, t ? XYZZ<Fp381>::identity() : xyzz_from_affine(load_affine_nc<Fp381>(mono, b)));
  store_xyzz<Fp381>(s_pts, kCellN + t, t ? xyzz_from_affine(load_affine_nc<Fp381>(mono, kCellN * (kCellN - t) + b)) : XYZZ<Fp381>::identity());
  __syncthreads();
  g1_dft_forward(s_pts, tw);
  store_affine<Fp381>(table, (size_t)kDft * b + t, xyzz_to_affine(load_xyzz<Fp381>(s_pts, t)));
  store_affine<Fp381>(table, (size_t)kDft * b + kCellN + t, xyzz_to_affine(load_xyzz<Fp381>(s_pts, kCellN + t)));
}

// One CTA per blob: the coefficients (the inverse NTT of kzg_cells_extend), then the 64 column DFTs, 16 columns per pass.
// hat[64 (128 blob + i) + b] = DFT(C_b)[brp7(i)] / (4096 * 128), canonical limbs: the scalars of MSM (blob, i), with the
// blob's 1/4096 and the inverse G1 DFT's 1/128 folded in.
__global__ void __launch_bounds__(kThreads, 1) kzg_fk20_columns(const uint8_t* __restrict__ blobs, const void* __restrict__ tw, void* __restrict__ hat) {
  extern __shared__ uint4 cells_smem[];
  uint4* cols = cells_smem + 2 * kN;
  load_blob(cells_smem, blobs + (size_t)blockIdx.x * kN * 32);
  ntt_inverse_brp(cells_smem, tw);
  const Fr381 ninv = tw_at(tw, kExtN);
  Fr381 scale = Fr381::mul(ninv, ninv);  // 1/4096^2 = 1/(4096 * 128) / 32
#pragma unroll 1
  for (int k = 0; k < 5; ++k) scale = Fr381::dbl(scale);
  void* out = (uint8_t*)hat + (size_t)blockIdx.x * kDft * kCellN * 32;
#pragma unroll 1
  for (uint32_t g = 0; g < kCellN; g += kColGroup) {
    for (uint32_t e = threadIdx.x; e < kColGroup * kDft; e += kThreads) {
      const uint32_t q = e / kDft, t = e % kDft;
      store_fe(cols, e, t < kCellN ? load_fe<Fr381>(cells_smem, kCellN * t + g + q) : Fr381::zero());
    }
    __syncthreads();
    for (uint32_t h = kDft / 2; h >= 1; h >>= 1) {
      const uint32_t step = kExtN / (2 * h);
#pragma unroll 1
      for (uint32_t e = threadIdx.x; e < kColGroup * kDft / 2; e += kThreads) {
        const uint32_t b = e % (kDft / 2), j = b & (h - 1), i0 = kDft * (e / (kDft / 2)) + 2 * b - j, i1 = i0 + h;
        const Fr381 u = load_fe<Fr381>(cols, i0), v = load_fe<Fr381>(cols, i1);
        store_fe(cols, i0, Fr381::add(u, v));
        store_fe(cols, i1, Fr381::mul(Fr381::sub(u, v), tw_at(tw, j * step)));
      }
      __syncthreads();
    }
    for (uint32_t e = threadIdx.x; e < kColGroup * kDft; e += kThreads) {
      const uint32_t q = e / kDft, i = e % kDft;
      store_fe(out, (size_t)kCellN * i + g + q, Fr381::mul(load_fe<Fr381>(cols, e), scale));
    }
    __syncthreads();
  }
}

B2_D Fp381 shfl_down_fp(const Fp381& a, uint32_t off) {
  Fp381 r;
#pragma unroll
  for (int k = 0; k < 12; ++k) r.v[k] = __shfl_down_sync(0xffffffffu, a.v[k], off);
  return r;
}

// One warp per MSM q = 128 blob + i: u[q] = sum_b hat[64 q + b] table[128 b + i], 64 terms.  Lane l takes b = 2l, 2l + 1
// with one shared doubling chain (Shamir's trick: P1, P2 or P1 + P2 per bit pair), then the warp sums its 32 lanes.
__global__ void __launch_bounds__(32 * kMsmWarps) kzg_fk20_msm(const void* __restrict__ table, const void* __restrict__ hat, size_t n_msm, void* __restrict__ u) {
  const size_t q = (size_t)blockIdx.x * kMsmWarps + threadIdx.x / 32;
  if (q >= n_msm) return;  // whole warps
  __shared__ uint4 s_pts[32 * kMsmWarps * 3 * 6];  // per thread P1, P2, P1 + P2 (96-byte affine), out of the registers
  const uint32_t lane = threadIdx.x % 32, i = (uint32_t)(q % kDft), b0 = 2 * lane, mine = 3 * threadIdx.x;
  {
    const Affine<Fp381> p1 = load_affine_nc<Fp381>(table, (size_t)kDft * b0 + i), p2 = load_affine_nc<Fp381>(table, (size_t)kDft * (b0 + 1) + i);
    XYZZ<Fp381> s12 = xyzz_from_affine(p1);
    xyzz_add_mixed(s12, p2.x, p2.y);
    store_affine<Fp381>(s_pts, mine, p1);
    store_affine<Fp381>(s_pts, mine + 1, p2);
    store_affine<Fp381>(s_pts, mine + 2, xyzz_to_affine(s12));
  }
  const Fr381 k1 = load_fe_nc<Fr381>(hat, kCellN * q + b0), k2 = load_fe_nc<Fr381>(hat, kCellN * q + b0 + 1);
  const Fp381* f = nullptr;
  XYZZ<Fp381> acc = XYZZ<Fp381>::identity();
#pragma unroll 1
  for (int bit = 254; bit >= 0; --bit) {
    acc = xyzz_dbl(acc);
    const uint32_t sel = ((k1.v[bit >> 5] >> (bit & 31)) & 1) | (((k2.v[bit >> 5] >> (bit & 31)) & 1) << 1);
    if (sel) {
      const uint32_t at = mine + sel - 1;
      xyzz_add_mixed(acc, load_field(s_pts, 2 * at, f), load_field(s_pts, 2 * at + 1, f));
    }
  }
#pragma unroll 1
  for (uint32_t off = 16; off; off >>= 1) {
    const XYZZ<Fp381> o = {shfl_down_fp(acc.x, off), shfl_down_fp(acc.y, off), shfl_down_fp(acc.zz, off), shfl_down_fp(acc.zzz, off)};
    xyzz_add(acc, o);
  }
  if (!lane) store_xyzz<Fp381>(u, q, acc);
}

// One CTA of 64 threads per blob: z = DFT^-1(u) (T_m = z[m]), v = (z[1] .. z[63], O ..), the 128 proofs DFT(v) in cell
// order, normalised and compressed (48 bytes each, blob-major)
__global__ void __launch_bounds__(kDft / 2, 1) kzg_fk20_proofs(const void* __restrict__ u, const void* __restrict__ tw, uint8_t* __restrict__ proofs) {
  __shared__ uint4 s_pts[kDft * 12];
  const uint32_t t = threadIdx.x;
  const size_t base = (size_t)kDft * blockIdx.x;
  store_xyzz<Fp381>(s_pts, t, load_xyzz<Fp381>(u, base + t));
  store_xyzz<Fp381>(s_pts, kCellN + t, load_xyzz<Fp381>(u, base + kCellN + t));
  __syncthreads();
  g1_dft_inverse(s_pts, tw);
  const XYZZ<Fp381> zt = t + 1 < kCellN ? load_xyzz<Fp381>(s_pts, t + 1) : XYZZ<Fp381>::identity();
  __syncthreads();
  store_xyzz<Fp381>(s_pts, t, zt);
  store_xyzz<Fp381>(s_pts, kCellN + t, XYZZ<Fp381>::identity());
  __syncthreads();
  g1_dft_forward(s_pts, tw);
  bls_g1_compress(proofs + 48 * (base + t), xyzz_to_affine(load_xyzz<Fp381>(s_pts, t)));
  bls_g1_compress(proofs + 48 * (base + kCellN + t), xyzz_to_affine(load_xyzz<Fp381>(s_pts, kCellN + t)));
}

// ---- cell recovery (c-kzg recover_cells_and_kzg_proofs) ------------------------------------------------------------
// Write p = sum_(j<64) X^j P_j(X^64), deg P_j < 64, so c_(64 m + j) = P_j[m].  Cell c holds I_c = p mod (X^64 - s_c) on
// its coset h_c <w_64> (point t at h_c w_64^brp6(t)), and I_c's coefficient j is P_j(s_c).  So per blob, from the first
// 64 given cells k (indices c_k, distinct, hence distinct s_k = w_128^brp7(c_k)):
//   E[k][j] = P_j(s_k) = NTT64^-1(cell k)[j] h_k^-j / 64           (64 inverse NTTs of size 64)
//   P_j[m]  = sum_k E[k][j] Q_k[m] / Z'(s_k)                     (Lagrange on the s_k: Z = prod (X - s_k), Q_k = Z / (X - s_k))
// one 64 x 64 by 64 x 64 product.  The forward NTT of the coefficients is the blob; tests/kzg_recover_ref.py restates
// this method with the same indexing and checks it against the consensus-spec recovery.

// One CTA per blob: blobs[b] (big-endian, as kzg_cells_extend takes it) from the first 64 of its given cells.  in: the
// given cells of every blob in order (big-endian, checked < r), offsets[b] its first, idx their cell indices.  Scratch
// per blob: lag (Q_k[m] at 64 k + m, Montgomery) and coef (c_i, canonical), 4096 elements each.
__global__ void __launch_bounds__(kThreads, 1) kzg_recover_blob(const uint8_t* __restrict__ in, const uint32_t* __restrict__ offsets,
                                                              const uint32_t* __restrict__ idx, const void* __restrict__ tw, void* lag,
                                                              void* coef, uint8_t* __restrict__ blobs) {
  extern __shared__ uint4 cells_smem[];
  __shared__ uint4 s_pt[2 * kCellN];        // s_k (Montgomery)
  __shared__ uint4 s_z[2 * (kCellN + 1)];   // Z's 65 coefficients (Montgomery)
  __shared__ uint4 s_w[2 * kCellN];         // 1 / (64 Z'(s_k)) (Montgomery)
  __shared__ uint32_t s_h[kCellN];          // brp7(c_k): h_k = w_8192^s_h[k]
  const uint32_t t = threadIdx.x, first = offsets[blockIdx.x];
  const uint8_t* given = in + (size_t)first * kCellN * 32;
  void* q = (uint8_t*)lag + (size_t)blockIdx.x * kN * 32;
  void* c = (uint8_t*)coef + (size_t)blockIdx.x * kN * 32;
  for (uint32_t i = t; i < kN; i += kThreads) store_fe(cells_smem, i, load_be32(given + 32 * i));
  if (t < kCellN) {
    s_h[t] = brp7(idx[first + t]);
    store_fe(s_pt, t, tw_at(tw, kCellN * s_h[t]));
  }
  if (t <= kCellN) store_fe(s_z, t, t ? Fr381::zero() : Fr381::one());
  __syncthreads();
  ntt_inverse_brp(cells_smem, tw, kCellN);
  // Z = prod_k (X - s_k): coefficient t of Z (X - s_k) is z[t - 1] - s_k z[t]
#pragma unroll 1
  for (uint32_t k = 0; k < kCellN; ++k) {
    Fr381 z;
    if (t <= kCellN) z = Fr381::sub(t ? load_fe<Fr381>(s_z, t - 1) : Fr381::zero(), Fr381::mul(load_fe<Fr381>(s_pt, k), load_fe<Fr381>(s_z, t)));
    __syncthreads();
    if (t <= kCellN) store_fe(s_z, t, z);
    __syncthreads();
  }
  // thread k: Q_k by synthetic division (Z is monic), and 1 / (64 Z'(s_k)) with Z'(s_k) = prod_(l != k) (s_k - s_l)
  if (t < kCellN) {
    const Fr381 s = load_fe<Fr381>(s_pt, t);
    Fr381 a = Fr381::one();
    store_fe(q, kCellN * t + kCellN - 1, a);
#pragma unroll 1
    for (uint32_t m = kCellN - 1; m; --m) {
      a = Fr381::add(load_fe<Fr381>(s_z, m), Fr381::mul(s, a));
      store_fe(q, kCellN * t + m - 1, a);
    }
    Fr381 d = Fr381::one();
#pragma unroll 1
    for (uint32_t l = 0; l < kCellN; ++l)
      if (l != t) d = Fr381::mul(d, Fr381::sub(s, load_fe<Fr381>(s_pt, l)));
#pragma unroll 1
    for (int k = 0; k < 6; ++k) d = Fr381::dbl(d);
    store_fe(s_w, t, Fr381::inv(d));
  }
  __syncthreads();
  // E[k][j] (canonical) in place
  for (uint32_t i = t; i < kN; i += kThreads) {
    const uint32_t k = i / kCellN, j = i % kCellN;
    const Fr381 unshift = Fr381::mul(tw_at(tw, (kExtN - s_h[k] * j) & (kExtN - 1)), load_fe<Fr381>(s_w, k));
    store_fe(cells_smem, i, Fr381::mul(load_fe<Fr381>(cells_smem, i), unshift));
  }
  __syncthreads();
  // c_(64 m + j) = sum_k E[k][j] Q_k[m]: a warp takes 32 consecutive j (one coalesced store) of one m
  const uint32_t j = t % kCellN;
#pragma unroll 1
  for (uint32_t m = t / kCellN; m < kCellN; m += kThreads / kCellN) {
    Fr381 acc = Fr381::zero();
#pragma unroll 1
    for (uint32_t k = 0; k < kCellN; ++k) acc = Fr381::add(acc, Fr381::mul(load_fe<Fr381>(cells_smem, kCellN * k + j), load_fe<Fr381>(q, kCellN * k + m)));
    store_fe(c, kCellN * m + j, acc);
  }
  __syncthreads();
  for (uint32_t i = t; i < kN; i += kThreads) store_fe(cells_smem, i, load_fe<Fr381>(c, i));
  __syncthreads();
  ntt_forward_brp(cells_smem, tw);
  uint8_t* blob = blobs + (size_t)blockIdx.x * kN * 32;
  for (uint32_t i = t; i < kN; i += kThreads) store_be32(blob + 32 * i, load_fe<Fr381>(cells_smem, i));
}

// One CTA per blob: bad[b] = the first position among the blob's given cells whose bytes differ from the rebuilt cell of
// its index in ext (n x 8192 x 32 bytes), or 0xffffffff when every given cell agrees
__global__ void __launch_bounds__(kThreads) kzg_recover_check(const uint8_t* __restrict__ in, const uint32_t* __restrict__ offsets,
                                                              const uint32_t* __restrict__ idx, const uint8_t* __restrict__ ext, uint32_t* __restrict__ bad) {
  __shared__ uint32_t s_bad;
  if (!threadIdx.x) s_bad = 0xffffffffu;
  __syncthreads();
  constexpr uint32_t kWords = kCellN * 32 / 16;  // 16-byte words per cell
  const uint32_t first = offsets[blockIdx.x], count = offsets[blockIdx.x + 1] - first;
  const uint4* given = reinterpret_cast<const uint4*>(in) + (size_t)first * kWords;
  const uint4* rebuilt = reinterpret_cast<const uint4*>(ext) + (size_t)blockIdx.x * kCells * kWords;
  for (uint32_t w = threadIdx.x; w < count * kWords; w += kThreads) {
    const uint32_t pos = w / kWords;
    const uint4 a = __ldg(given + w), e = __ldg(rebuilt + idx[first + pos] * kWords + w % kWords);
    if (a.x != e.x || a.y != e.y || a.z != e.z || a.w != e.w) atomicMin(&s_bad, pos);
  }
  __syncthreads();
  if (!threadIdx.x) bad[blockIdx.x] = s_bad;
}

// the twiddle table, built on first use
int cells_tw(b200zk_ctx* ctx, cudaStream_t st, const void** tw) {
  B2_TRY(once_table(ctx, ctx->kzg_cells_tw, (kExtN + 1) * 32, st, [&](void* t) -> int {
    B2_LAUNCH(ctx, kzg_cells_tw_build, (kExtN + 256) / 256, 256, 0, st, t);
    return B200ZK_OK;
  }, tw));
  if (!ctx->attr_kzg_cells) {
    B2_CUDA(ctx, cudaFuncSetAttribute(kzg_cells_extend, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
    B2_CUDA(ctx, cudaFuncSetAttribute(kzg_cells_interp, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
    B2_CUDA(ctx, cudaFuncSetAttribute(kzg_cells_interp_eval, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
    B2_CUDA(ctx, cudaFuncSetAttribute(kzg_fk20_columns, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kColSmem));
    B2_CUDA(ctx, cudaFuncSetAttribute(kzg_recover_blob, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
    B2_CUDA(ctx, cudaFuncSetAttribute(kzg_vcells_columns, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmem));
    ctx->attr_kzg_cells = true;
  }
  return B200ZK_OK;
}

// the FK20 table of a monomial setup, built on the handle's first cell-proof call
int fk20_table(b200zk_ctx* ctx, BasesEntry& e, const void* tw, cudaStream_t st, const void** table) {
  return once_table(ctx, e.fk20, (size_t)kCellN * kDft * 96, st, [&](void* t) -> int {
    B2_LAUNCH(ctx, kzg_fk20_table, kCellN, kDft / 2, 0, st, (const void*)e.d.p, tw, t);
    return B200ZK_OK;
  }, table);
}

// the 128 proofs of each of n blobs (d_blobs, checked < r) by FK20 into d_proofs; scratch hat n x 128 x 64 x 32 bytes, u
// n x 128 x 192 bytes
int fk20_run(b200zk_ctx* ctx, BasesEntry& mono, const uint8_t* d_blobs, size_t n, void* d_hat, void* d_u, uint8_t* d_proofs, cudaStream_t st) {
  const void *tw = nullptr, *table = nullptr;
  B2_TRY(cells_tw(ctx, st, &tw));
  B2_TRY(fk20_table(ctx, mono, tw, st, &table));
  B2_LAUNCH(ctx, kzg_fk20_columns, (unsigned)n, kThreads, kColSmem, st, d_blobs, tw, d_hat);
  const size_t n_msm = n * kDft;
  B2_LAUNCH(ctx, kzg_fk20_msm, (unsigned)((n_msm + kMsmWarps - 1) / kMsmWarps), 32 * kMsmWarps, 0, st, table, (const void*)d_hat, n_msm, d_u);
  B2_LAUNCH(ctx, kzg_fk20_proofs, (unsigned)n, kDft / 2, 0, st, (const void*)d_u, tw, d_proofs);
  return B200ZK_OK;
}

// host checks of a recovery batch: offsets, 64..128 cells per blob, indices < 128 and distinct within a blob (status 2)
int check_recover_indices(b200zk_ctx* ctx, const uint32_t* offsets, const uint64_t* indices, size_t n, const char* what) {
  B2_TRY(check_offsets(ctx, offsets, n, what));
  char msg[192];
  for (size_t b = 0; b < n; ++b) {
    const uint32_t count = offsets[b + 1] - offsets[b];
    if (count < kCellN || count > kCells) {
      snprintf(msg, sizeof msg, "%s: blob %zu has %u cells; recovery takes 64 to 128", what, b, count);
      return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, msg);
    }
    bool seen[kCells] = {};
    for (uint32_t k = 0; k < count; ++k) {
      const uint64_t c = indices[offsets[b] + k];
      if (c >= kCells || seen[c]) {
        snprintf(msg, sizeof msg, "%s: blob %zu, cell %u: index %llu is %s", what, b, k, (unsigned long long)c, c >= kCells ? "not below 128" : "repeated");
        return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, msg);
      }
      seen[c] = true;
    }
  }
  return B200ZK_OK;
}

}  // namespace

int kzg_cells_run(b200zk_ctx* ctx, const uint8_t* d_blobs, size_t n, uint8_t* d_cells, cudaStream_t st) {
  const void* tw = nullptr;
  B2_TRY(cells_tw(ctx, st, &tw));
  B2_LAUNCH(ctx, kzg_cells_extend, (unsigned)n, kThreads, kSmem, st, d_blobs, tw, d_cells);
  return B200ZK_OK;
}

int kzg_cell_scalars_run(b200zk_ctx* ctx, const uint8_t* d_blobs, size_t n, const uint8_t* d_r_be, void* d_weights, void* d_partial,
                         void* d_s_proof, void* d_s_lin, void* d_s_setup, cudaStream_t st) {
  const void* tw = nullptr;
  B2_TRY(cells_tw(ctx, st, &tw));
  B2_LAUNCH(ctx, kzg_cells_weights, 1, 96, 0, st, d_r_be, tw, d_weights);
  B2_LAUNCH(ctx, kzg_cells_interp, (unsigned)n, kThreads, kSmem, st, d_blobs, tw, (const void*)d_weights, d_partial);
  B2_LAUNCH(ctx, kzg_cells_interp_eval, 1, kThreads, kSmem, st, (const void*)d_partial, n, tw, d_s_setup);
  B2_LAUNCH(ctx, kzg_cells_scalars, (unsigned)(((kCells + 1) * n + 255) / 256), 256, 0, st, tw, (const void*)d_weights, n, d_s_proof, d_s_lin);
  return B200ZK_OK;
}

int kzg_vcells_scalars_run(b200zk_ctx* ctx, const uint8_t* d_cells, const VCellsMeta& m, const uint8_t* d_r_be, void* d_rpow, void* d_partial,
                           void* d_s_proof, void* d_s_lin, void* d_s_setup, cudaStream_t st) {
  const void* tw = nullptr;
  B2_TRY(cells_tw(ctx, st, &tw));
  B2_LAUNCH(ctx, kzg_vcells_powers, (unsigned)((m.n + 255) / 256), 256, 0, st, d_r_be, tw, m.idx, m.n, m.n_commit, d_rpow, d_s_proof, d_s_lin);
  B2_LAUNCH(ctx, kzg_vcells_weights, (unsigned)((m.n_commit + 255) / 256), 256, 0, st, m.commit_off, m.by_commit, m.n_commit, (const void*)d_s_proof, d_s_lin);
  B2_LAUNCH(ctx, kzg_vcells_columns, (unsigned)((m.n_cols + kCellN - 1) / kCellN), kThreads, kSmem, st, d_cells, (const void*)d_rpow, m.column_off,
            m.by_column, m.columns, m.n_cols, tw, d_partial);
  B2_LAUNCH(ctx, kzg_cells_interp_eval, 1, kThreads, kSmem, st, (const void*)d_partial, m.n_cols, tw, d_s_setup);
  return B200ZK_OK;
}

}  // namespace b200zk

using namespace b200zk;

extern "C" {

int b200zk_kzg_compute_cells(b200zk_ctx* ctx, const uint8_t* blobs, size_t n_blobs, uint8_t* cells) {
  static const char* what = "kzg_compute_cells";
  if (!ctx || (n_blobs && (!blobs || !cells))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_compute_cells: null argument");
  NvtxRange nvtx("b200zk:kzg_compute_cells");
  DeviceGuard guard(ctx);
  if (!n_blobs) return B200ZK_OK;
  cudaStream_t st = ctx->stream;
  uint8_t *d_blobs, *d_cells;
  B2_TRY(carve(ctx, ctx->ws_kzg, [&](Carve& c) {
    d_blobs = c.take<uint8_t>(n_blobs * kN * 32); d_cells = c.take<uint8_t>(n_blobs * kExtN * 32);
  }));
  B2_CUDA(ctx, cudaMemcpyAsync(d_blobs, blobs, n_blobs * kN * 32, cudaMemcpyHostToDevice, st));
  B2_TRY(check_blobs(ctx, d_blobs, n_blobs, 0, st, what));
  B2_TRY(kzg_cells_run(ctx, d_blobs, n_blobs, d_cells, st));
  B2_CUDA(ctx, cudaMemcpyAsync(cells, d_cells, n_blobs * kExtN * 32, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

int b200zk_kzg_blob_to_commitment_and_cell_proofs(b200zk_ctx* ctx, uint64_t g1_lagrange, uint64_t g1_monomial, const uint8_t* blobs, size_t n_blobs,
                                                  uint8_t* commitments, uint8_t* proofs) {
  static const char* what = "kzg_blob_to_commitment_and_cell_proofs";
  if (!ctx || (n_blobs && (!blobs || !commitments || !proofs))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_blob_to_commitment_and_cell_proofs: null argument");
  NvtxRange nvtx("b200zk:kzg_blob_to_commitment_and_cell_proofs");
  DeviceGuard guard(ctx);
  BasesEntry *lag = nullptr, *mono = nullptr;
  B2_TRY(kzg_setup(ctx, g1_lagrange, "kzg_blob_to_commitment_and_cell_proofs (g1_lagrange)", &lag));
  B2_TRY(kzg_setup(ctx, g1_monomial, "kzg_blob_to_commitment_and_cell_proofs (g1_monomial)", &mono));
  if (!n_blobs) return B200ZK_OK;
  cudaStream_t st = ctx->stream;
  uint8_t *d_blobs, *d_hat, *d_u, *d_partials, *d_enc, *d_proofs;
  B2_TRY(carve(ctx, ctx->ws_kzg, [&](Carve& c) {
    d_blobs = c.take<uint8_t>(n_blobs * kN * 32);
    d_hat = c.take<uint8_t>(n_blobs * kDft * kCellN * 32);
    d_u = c.take<uint8_t>(n_blobs * kDft * 192);
    d_partials = c.take<uint8_t>(n_blobs * 192);
    d_enc = c.take<uint8_t>(n_blobs * 128);
    d_proofs = c.take<uint8_t>(n_blobs * kCells * 48);
  }));
  B2_CUDA(ctx, cudaMemcpyAsync(d_blobs, blobs, n_blobs * kN * 32, cudaMemcpyHostToDevice, st));
  B2_TRY(check_blobs(ctx, d_blobs, n_blobs, 0, st, what));
  B2_TRY(fk20_run(ctx, *mono, d_blobs, n_blobs, d_hat, d_u, d_proofs, st));
  B2_TRY(kzg_msms(ctx, *lag, d_blobs, n_blobs, B200ZK_SCALARS_BE, d_partials, d_enc, st));
  std::vector<uint8_t> enc(n_blobs * 128);
  B2_CUDA(ctx, cudaMemcpyAsync(enc.data(), d_enc, enc.size(), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(proofs, d_proofs, n_blobs * kCells * 48, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  for (size_t b = 0; b < n_blobs; ++b) memcpy(commitments + 48 * b, &enc[128 * b], 48);
  return B200ZK_OK;
}

int b200zk_kzg_recover_cells_and_cell_proofs(b200zk_ctx* ctx, uint64_t g1_monomial, const uint32_t* cell_offsets, const uint64_t* cell_indices,
                                             const uint8_t* cells, size_t n_blobs, uint8_t* cells_out, uint8_t* proofs_out) {
  static const char* what = "kzg_recover_cells_and_cell_proofs";
  if (!ctx || (n_blobs && (!cell_offsets || !cell_indices || !cells || !cells_out || !proofs_out)))
    return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_recover_cells_and_cell_proofs: null argument");
  NvtxRange nvtx("b200zk:kzg_recover_cells_and_cell_proofs");
  DeviceGuard guard(ctx);
  BasesEntry* mono = nullptr;
  B2_TRY(kzg_setup(ctx, g1_monomial, "kzg_recover_cells_and_cell_proofs (g1_monomial)", &mono));
  if (!n_blobs) return B200ZK_OK;
  B2_TRY(check_recover_indices(ctx, cell_offsets, cell_indices, n_blobs, what));
  const size_t total = cell_offsets[n_blobs];
  std::vector<uint32_t> meta(n_blobs + 1 + total);  // offsets, then the indices
  for (size_t b = 0; b <= n_blobs; ++b) meta[b] = cell_offsets[b];
  for (size_t k = 0; k < total; ++k) meta[n_blobs + 1 + k] = (uint32_t)cell_indices[k];
  cudaStream_t st = ctx->stream;
  const size_t cells_bytes = n_blobs * kExtN * 32, proofs_bytes = n_blobs * kCells * 48;
  uint8_t *d_in, *d_lag, *d_coef, *d_blobs, *d_hat, *d_u, *d_out;
  uint32_t* d_meta;
  B2_TRY(carve(ctx, ctx->ws_kzg, [&](Carve& c) {
    d_in = c.take<uint8_t>(total * kCellN * 32);
    d_meta = c.take<uint32_t>(meta.size());
    d_lag = c.take<uint8_t>(n_blobs * kN * 32);
    d_coef = c.take<uint8_t>(n_blobs * kN * 32);
    d_blobs = c.take<uint8_t>(n_blobs * kN * 32);
    d_hat = c.take<uint8_t>(n_blobs * kDft * kCellN * 32);
    d_u = c.take<uint8_t>(n_blobs * kDft * 192);
    d_out = c.take<uint8_t>(cells_bytes + proofs_bytes + n_blobs * 4);  // cells | proofs | bad: one copy back
  }));
  uint8_t* d_proofs = d_out + cells_bytes;
  uint32_t* d_bad = reinterpret_cast<uint32_t*>(d_proofs + proofs_bytes);
  B2_CUDA(ctx, cudaMemcpyAsync(d_in, cells, total * kCellN * 32, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(d_meta, meta.data(), meta.size() * 4, cudaMemcpyHostToDevice, st));
  size_t bad = total * kCellN;
  B2_TRY(bls_scalars_check(ctx, d_in, total * kCellN, true, st, &bad));
  if (bad < total * kCellN) {
    const size_t pos = bad / kCellN, b = std::upper_bound(cell_offsets, cell_offsets + n_blobs + 1, (uint32_t)pos) - cell_offsets - 1;
    char msg[192];
    snprintf(msg, sizeof msg, "%s: blob %zu, cell %zu, element %zu is >= the BLS12-381 group order", what, b, pos - cell_offsets[b], bad % kCellN);
    return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, msg);
  }
  const uint32_t* d_offsets = d_meta;
  const uint32_t* d_idx = d_meta + n_blobs + 1;
  const void* tw = nullptr;
  B2_TRY(cells_tw(ctx, st, &tw));
  B2_LAUNCH(ctx, kzg_recover_blob, (unsigned)n_blobs, kThreads, kSmem, st, (const uint8_t*)d_in, d_offsets, d_idx, tw, (void*)d_lag, (void*)d_coef, d_blobs);
  B2_TRY(kzg_cells_run(ctx, d_blobs, n_blobs, d_out, st));
  B2_LAUNCH(ctx, kzg_recover_check, (unsigned)n_blobs, kThreads, 0, st, (const uint8_t*)d_in, d_offsets, d_idx, (const uint8_t*)d_out, d_bad);
  B2_TRY(fk20_run(ctx, *mono, d_blobs, n_blobs, d_hat, d_u, d_proofs, st));
  std::vector<uint8_t> h(cells_bytes + proofs_bytes + n_blobs * 4);
  B2_CUDA(ctx, cudaMemcpyAsync(h.data(), d_out, h.size(), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  for (size_t b = 0; b < n_blobs; ++b) {
    uint32_t pos;
    memcpy(&pos, &h[cells_bytes + proofs_bytes + 4 * b], 4);
    if (pos == 0xffffffffu) continue;
    char msg[224];
    snprintf(msg, sizeof msg, "%s: blob %zu, cell %u (index %llu) does not lie on the polynomial of its first 64 cells", what, b, pos,
             (unsigned long long)cell_indices[cell_offsets[b] + pos]);
    return fail(ctx, B200ZK_ERR_NOT_ON_CURVE, msg);
  }
  memcpy(cells_out, h.data(), cells_bytes);
  memcpy(proofs_out, h.data() + cells_bytes, proofs_bytes);
  return B200ZK_OK;
}

}  // extern "C"
