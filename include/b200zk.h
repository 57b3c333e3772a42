/* b200zk.h -- frozen C ABI of libb200zk.so, the H100 (sm_90a) BN254 MSM + Fr NTT backend.
 *
 * This is the drop-in boundary for ethrex's L2 prover hot path (SURVEY.md section 8b): the entry points a
 * `crates/prover/src/backend/b200.rs` ProverBackend implementation binds through `unsafe extern "C"`
 * (the binding a maintainer adds is shown in INTEGRATION.md and rust/b200zk-sys/src/lib.rs).
 *
 * Conventions follow the in-tree C-ABI precedent
 *   /root/reference/crates/guest-program/src/crypto/zisk.rs:5-64   (declarations)
 *   /root/reference/crates/guest-program/src/crypto/zisk.rs:144-172 (status codes 0/1/2/3)
 * i.e. caller-owned buffers, plain pointers and sizes, small integer status, nothing allocated across the
 * boundary except opaque handles.  No torch / CUDA types appear in any signature: device pointers and
 * streams travel as `void*` (a `cudaStream_t` is a pointer).
 *
 * Byte formats
 *   "BE"      32-byte big-endian canonical field elements, the EIP-196/197 wire format of
 *             /root/reference/crates/common/crypto/provider.rs:201-330: G1 = x|y (64 B), (0,0) = identity;
 *             G2 = x_im|x_re|y_im|y_re (128 B); coordinates >= p are rejected like
 *             /root/reference/crates/vm/levm/src/precompiles.rs:801-820.
 *   "native"  little-endian limbs (bytes of 4 x u64 == 8 x u32 on a little-endian host).  Field elements of
 *             points and NTT data are in Montgomery form with R = 2^256 -- the in-memory form of ark-ff
 *             0.5.0 Fp256<MontBackend> that the SNARK wrap behind ProofFormat::Groth16
 *             (/root/reference/crates/prover/src/backend/sp1.rs:97-134, risc0.rs:24-29) holds its proving
 *             key in.  G1 affine = x|y (64 B), G2 affine = x.c0|x.c1|y.c0|y.c1 (128 B), (0,..,0) = identity.
 *             Scalars are canonical (non-Montgomery) 256-bit integers (ark `into_bigint()`), reduced mod r by
 *             the library, unless B200ZK_SCALARS_MONT is set.
 *
 * Semantics
 *   MSM  = ark_ec::VariableBaseMSM::msm (ark-ec 0.5.0, /root/reference/Cargo.lock:978): sum_i s_i * P_i,
 *          returned as the affine point -- the value is algorithm independent, so "bit exact" means equal
 *          (x, y).
 *   NTT  = ark_poly::Radix2EvaluationDomain (ark-poly 0.5.0, /root/reference/Cargo.lock:1140), equal to
 *          gnark-crypto's bn254 fr/fft: natural order in and out, out[k] = sum_j a[j] w^{jk},
 *          w = 5^((r-1)/2^28)^(2^(28-log_n)); inverse uses w^-1 and scales by n^-1; coset pre-multiplies a[j]
 *          by h^j (forward) / post-multiplies by h^-j (inverse), h = 5 unless given.
 *
 * Threading and streams
 *   Every entry point switches to the context's device for the duration of the call (and restores the caller's),
 *   so a context may be used from any thread and next to contexts on other devices.  A context owns ONE set of
 *   grow-only scratch buffers: drive it from one stream at a time (or order the streams with events yourself).
 *   Cached tables (NTT twiddles, coset powers) carry a build event that consumers on other streams wait on.
 *
 * There is NO CPU fallback anywhere behind this interface: without a CUDA device b200zk_init fails with
 * B200ZK_ERR_NO_DEVICE and every other call fails with B200ZK_ERR_INVALID_ARG on the NULL context.
 */
#ifndef B200ZK_H
#define B200ZK_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200ZK_ABI_VERSION 2 /* v2: async MSM forms append a 4-byte is-infinity word; groth16 + ntt-root entry points */

typedef struct b200zk_ctx b200zk_ctx;

/* status codes: 0..3 are the ZisK table (zisk.rs:144-172); the rest are this library's own failures */
enum {
  B200ZK_OK = 0,
  B200ZK_OK_INFINITY = 1,       /* success, result is the identity */
  B200ZK_ERR_NOT_IN_FIELD = 2,  /* a BE coordinate is >= p */
  B200ZK_ERR_NOT_ON_CURVE = 3,  /* a BE point does not satisfy the curve equation */
  B200ZK_ERR_INVALID_ARG = 4,
  B200ZK_ERR_CUDA = 5,
  B200ZK_ERR_NO_DEVICE = 6,
  B200ZK_ERR_OOM = 7,
  B200ZK_ERR_UNSUPPORTED = 8
};

/* flags */
enum {
  B200ZK_POINTS_BE = 1u << 0,       /* points are EIP-196/197 big-endian bytes (validated); default native */
  B200ZK_SCALARS_BE = 1u << 1,      /* scalars are 32-byte big-endian; default little-endian limbs */
  B200ZK_SCALARS_MONT = 1u << 2,    /* scalars are Montgomery-form limbs (ark Fr in-memory form) */
  B200ZK_OUT_NATIVE = 1u << 3,      /* MSM result as native affine limbs instead of BE bytes */
  B200ZK_NTT_INVERSE = 1u << 4,
  B200ZK_NTT_COSET = 1u << 5,
  B200ZK_NTT_CANONICAL = 1u << 6,   /* NTT data are canonical little-endian limbs (converted on device) */
  B200ZK_NTT_BE = 1u << 7,          /* NTT data are 32-byte big-endian canonical values */
  B200ZK_G16_INPUTS_DEVICE = 1u << 8, /* b200zk_groth16_commit*: witness and evaluation buffers are DEVICE pointers (used in place) */
  B200ZK_G16_H_COEFFS = 1u << 9,    /* b200zk_groth16_commit*: a_evals already holds the quotient's coefficients (Montgomery); skip the NTTs */
  B200ZK_SCALARS_RAW = 1u << 10,    /* internal to the BLS12-381 calls (scalars range-checked, not reduced); every BN254 MSM entry point
                                       refuses it with B200ZK_ERR_INVALID_ARG */
  B200ZK_POINTS_COMPRESSED = 1u << 11 /* BLS12-381 G1 points in the 48-byte compressed ZCash / IETF format (the trusted setup's form) */
};

/* ---- lifecycle (ProverBackend::new / process-global OnceLock, cf. sp1.rs:30,93-95) ------------------- */
int b200zk_abi_version(void);
int b200zk_device_count(void);
int b200zk_init(int device, b200zk_ctx** out);
void b200zk_destroy(b200zk_ctx* ctx);
const char* b200zk_strerror(int status);
const char* b200zk_last_error(const b200zk_ctx* ctx); /* detail of the last failure on this context */
/* number of kernels this context has launched since init (bench.py's gpu_launches claim) */
uint64_t b200zk_launch_count(const b200zk_ctx* ctx);
int b200zk_synchronize(b200zk_ctx* ctx);

/* ---- host-buffer entry points: what the Rust backend calls.  Copies are part of the call. -------------- */
/* replaces ark_ec::VariableBaseMSM::msm for G1Affine / G2Affine (SURVEY.md 8a rows a6, a7) */
int b200zk_g1_msm(b200zk_ctx* ctx, const void* points, const void* scalars, size_t n, uint32_t flags,
                  uint8_t out[64]);
int b200zk_g2_msm(b200zk_ctx* ctx, const void* points, const void* scalars, size_t n, uint32_t flags,
                  uint8_t out[128]);
/* replaces ark_poly::Radix2EvaluationDomain::{fft,ifft,coset_fft,coset_ifft}_in_place (row a8);
 * n = 2^log_n elements of 32 bytes, transformed in place in the caller's buffer. coset_gen: 32-byte
 * canonical value in the same endianness family as the data (LE limbs, or BE with B200ZK_NTT_BE); NULL = 5 */
int b200zk_fr_ntt(b200zk_ctx* ctx, void* data, uint32_t log_n, uint32_t flags, const uint8_t* coset_gen);

/* ---- resident bases: the proving key (SRS) lives in HBM across proofs ---------------------------------- */
int b200zk_g1_bases_upload(b200zk_ctx* ctx, const void* points, size_t n, uint32_t flags, uint64_t* handle);
int b200zk_g2_bases_upload(b200zk_ctx* ctx, const void* points, size_t n, uint32_t flags, uint64_t* handle);
/* same, from points already in device memory (native format); the library keeps its own copy */
int b200zk_g1_bases_from_device(b200zk_ctx* ctx, const void* d_points, size_t n, void* stream, uint64_t* handle);
int b200zk_g2_bases_from_device(b200zk_ctx* ctx, const void* d_points, size_t n, void* stream, uint64_t* handle);
/* One-off, when the proving key is loaded: replace the resident bases by a table of their window multiples
 * 2^(c*w) * P_i, w = 0..ceil(255/c)-1 (W times the memory).  All windows then share ONE bucket set: larger
 * windows pay off (c = 22 -> 12 n additions instead of 15 n at 2^24) and the final Horner pass disappears.
 * window_bits = 0 picks c from n.  Results are unchanged (same group element). */
int b200zk_bases_precompute(b200zk_ctx* ctx, uint64_t handle, uint32_t window_bits);
int b200zk_bases_free(b200zk_ctx* ctx, uint64_t handle);
/* MSM of the first n resident bases against host scalars */
int b200zk_g1_msm_resident(b200zk_ctx* ctx, uint64_t handle, const void* scalars, size_t n, uint32_t flags,
                           uint8_t out[64]);
int b200zk_g2_msm_resident(b200zk_ctx* ctx, uint64_t handle, const void* scalars, size_t n, uint32_t flags,
                           uint8_t out[128]);
/* resident bases against scalars already in device memory (`stream` as for the *_device calls below) */
int b200zk_g1_msm_resident_device(b200zk_ctx* ctx, uint64_t handle, const void* d_scalars, size_t n,
                                  uint32_t flags, void* stream, uint8_t out[64]);
int b200zk_g2_msm_resident_device(b200zk_ctx* ctx, uint64_t handle, const void* d_scalars, size_t n,
                                  uint32_t flags, void* stream, uint8_t out[128]);

/* ---- device-pointer entry points: inputs already in HBM (native formats only) ------------------------- */
/* `stream`: a cudaStream_t passed as void*; NULL = the context's own (non-blocking) stream, so pass
 * cudaStreamLegacy ((void*)0x1) to mean the legacy default stream.  The *_device calls enqueue
 * every kernel on that stream, then copy the 64/128-byte result to `out` and wait for it. */
int b200zk_g1_msm_device(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n,
                         uint32_t flags, void* stream, uint8_t out[64]);
int b200zk_g2_msm_device(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n,
                         uint32_t flags, void* stream, uint8_t out[128]);
/* fully asynchronous forms: the encoded result (BE or native per flags) is written to device memory, followed by a
 * 32-bit word that is 1 when the result is the identity (what the synchronous forms return as status 1):
 * d_out68 = 64 + 4 bytes, d_out132 = 128 + 4 bytes */
int b200zk_g1_msm_device_async(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n,
                               uint32_t flags, void* stream, void* d_out68);
int b200zk_g2_msm_device_async(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n,
                               uint32_t flags, void* stream, void* d_out132);
int b200zk_fr_ntt_device(b200zk_ctx* ctx, void* d_data, uint32_t log_n, uint32_t flags,
                         const uint8_t* coset_gen, void* stream);
/* The primitive 2^28-th root of unity g of Fr that every domain generator derives from (w_n = g^(2^(28-log_n))) is a
 * parameter of the context (SURVEY.md section 8c).  root_le = canonical little-endian 32 bytes, NULL = back to the
 * default.  Rejected with B200ZK_ERR_INVALID_ARG unless g^(2^28) = 1 and g^(2^27) != 1.
 *   preset 0  ark-poly 0.5.0 / gnark-crypto bn254 fr:  5^((r-1)/2^28) = 0x2a3c09f0a58a7e8500e0a7eb8ef62abc402d111e41112ed49bd61b6e725b19f0
 *             (the SP1 / RISC0 Groth16 wraps, /root/reference/crates/prover/src/backend/sp1.rs:97-134, risc0.rs:24-29)   [default]
 *   preset 1  halo2curves-axiom 0.7.2 bn256::Fr:       7^((r-1)/2^28) = 0x03ddb9f5166d18b798865ea93dd31f743215cf6dd39329c8d34f1ed960c37c9c
 *             (the OpenVM halo2-KZG wrap, /root/reference/crates/prover/src/backend/openvm.rs:52-56) */
int b200zk_set_ntt_root(b200zk_ctx* ctx, const uint8_t* root_le);
int b200zk_ntt_root_preset(int preset, uint8_t root_le_out[32]);

/* ---- multi-GPU: one process per GPU, point-split MSM (SURVEY.md 8e) ------------------------------------ */
/* Each rank reduces its shard to ONE partial sum in extended-Jacobian XYZZ form (G1: 128 B, G2: 256 B,
 * native Montgomery limbs) left in device memory; the host side all-gathers the partials over NCCL and
 * every rank folds them with b200zk_g{1,2}_fold_partials_device -- NCCL has no elliptic-curve reduce op, so
 * this pair is the "allreduce of partial sums". */
int b200zk_g1_msm_partial_device(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n,
                                 uint32_t flags, void* stream, void* d_partial128);
int b200zk_g2_msm_partial_device(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n,
                                 uint32_t flags, void* stream, void* d_partial256);
/* same, over resident (possibly precomputed) bases */
int b200zk_g1_msm_partial_resident_device(b200zk_ctx* ctx, uint64_t handle, const void* d_scalars, size_t n,
                                          uint32_t flags, void* stream, void* d_partial128);
int b200zk_g2_msm_partial_resident_device(b200zk_ctx* ctx, uint64_t handle, const void* d_scalars, size_t n,
                                          uint32_t flags, void* stream, void* d_partial256);
/* same, with the shard's scalars in (pinned) HOST memory: the upload is pipelined with the accumulation */
int b200zk_g1_msm_partial_resident(b200zk_ctx* ctx, uint64_t handle, const void* scalars, size_t n, uint32_t flags,
                                   void* stream, void* d_partial128);
int b200zk_g2_msm_partial_resident(b200zk_ctx* ctx, uint64_t handle, const void* scalars, size_t n, uint32_t flags,
                                   void* stream, void* d_partial256);
int b200zk_g1_fold_partials_device(b200zk_ctx* ctx, const void* d_partials, size_t count, uint32_t flags,
                                   void* stream, uint8_t out[64]);
int b200zk_g2_fold_partials_device(b200zk_ctx* ctx, const void* d_partials, size_t count, uint32_t flags,
                                   void* stream, uint8_t out[128]);

/* ---- device utilities (format conversion, synthetic workloads; used by tests and bench.py) ------------- */
/* canonical LE limbs <-> Montgomery limbs, in place in device memory; which = 0 for Fq, 1 for Fr */
int b200zk_field_to_mont_device(b200zk_ctx* ctx, void* d_data, size_t n, int which, void* stream);
int b200zk_field_from_mont_device(b200zk_ctx* ctx, void* d_data, size_t n, int which, void* stream);
/* out[i] = a[i] * b[i] (Montgomery product), the field core exposed for parity tests and microbenchmarks;
 * `repeat` > 1 chains out = out * b that many times (throughput measurement).
 * which: 0 = Fq, 1 = Fr; +2 = the dedicated squaring instead (out = a^2, chained: a^(2^repeat); d_b is read but unused) */
int b200zk_field_mul_device(b200zk_ctx* ctx, const void* d_a, const void* d_b, void* d_out, size_t n,
                            int which, uint32_t repeat, void* stream);
/* out[i] = (a[i]*b[i] - c[i]) * zinv over Fr (Montgomery data; zinv canonical LE): the pointwise step of the
 * Groth16 quotient H = (A*B - C)/Z_H evaluated on a coset, where Z_H is the constant h^n - 1 */
int b200zk_fr_quotient_device(b200zk_ctx* ctx, const void* d_a, const void* d_b, const void* d_c, void* d_out,
                              size_t n, const uint8_t zinv[32], void* stream);
/* counter-based splitmix64 scalars: element i = reduce_mod_r(4 outputs of state seed + 4*(start+i)*golden)
 * (SURVEY.md 8d); canonical limbs, or Montgomery with B200ZK_SCALARS_MONT */
int b200zk_fr_random_device(b200zk_ctx* ctx, void* d_out, size_t n, uint64_t seed, uint64_t start,
                            uint32_t flags, void* stream);
/* synthetic base chain P_i = (k + i*d) * G for i in [start, start+n) (native affine);
 * k, d: canonical LE 32-byte scalars */
int b200zk_g1_chain_device(b200zk_ctx* ctx, void* d_out, size_t start, size_t n, const uint8_t k[32],
                           const uint8_t d[32], void* stream);
int b200zk_g2_chain_device(b200zk_ctx* ctx, void* d_out, size_t start, size_t n, const uint8_t k[32],
                           const uint8_t d[32], void* stream);
/* on-curve check of n native affine points; *bad_index = first offending index or n */
int b200zk_g1_check_device(b200zk_ctx* ctx, const void* d_points, size_t n, void* stream, size_t* bad_index);
int b200zk_g2_check_device(b200zk_ctx* ctx, const void* d_points, size_t n, void* stream, size_t* bad_index);

/* tuning knobs (0 = automatic): window bits for the next MSM calls on this context */
int b200zk_set_msm_window(b200zk_ctx* ctx, uint32_t c);
/* chunks of the pipelined MSM schedule (sort of chunk k+1 overlaps the accumulation of chunk k); 0 = automatic
 * (4 from 2^22 points), 1 = one shot */
int b200zk_set_msm_chunks(b200zk_ctx* ctx, uint32_t chunks);
/* rounds of batched-affine pair summing run before the bucket accumulation (0..4; negative = automatic) */
int b200zk_set_msm_pair_rounds(b200zk_ctx* ctx, int rounds);
/* per-phase device time of the last *_device MSM call, in milliseconds:
 * [0] digit histogram, [1] scan, [2] scatter, [3] bucket accumulation, [4] bucket reduction, [5] final */
int b200zk_last_msm_phase_ms(b200zk_ctx* ctx, float out_ms[6]);
int b200zk_set_profiling(b200zk_ctx* ctx, int enabled);

/* Several resident-base MSMs over ONE scalar vector -- Groth16's [A]1, [B]1, [B]2 and [L]1 all multiply the witness
 * (the prove step behind crates/prover/src/backend/sp1.rs:97-134 / risc0.rs:71-82).  The scalar-dependent half of
 * the MSM (digit recoding, bucket histogram, scan, scatter: ~15 % of a 2^24 MSM) runs once and is shared; G1 and G2
 * handles may be mixed.  All handles must have been precomputed with the same window (or none of them) and, when
 * precomputed, hold the same number of points.  out: `count` slots of 128 bytes (a G1 result uses the first 64);
 * status[i] = 0, or 1 when result i is the identity.  Device scalars, like b200zk_g1_msm_resident_device. */
int b200zk_msm_multi_resident_device(b200zk_ctx* ctx, const uint64_t* handles, size_t count, const void* d_scalars, size_t n,
                                     uint32_t flags, void* stream, uint8_t* out /* count*128 */, int* status /* count */);

/* ---- the Groth16 prove arithmetic as one call (SURVEY.md section 8b / 8f row 1) --------------------------------------
 * What the SNARK wrap behind ProofFormat::Groth16 computes after witness generation
 * (crates/prover/src/backend/sp1.rs:97-134 -> gnark groth16.Prove; risc0.rs:24-29,71-82 -> risc0-groth16), over a
 * proving key that lives in HBM (b200zk_g{1,2}_bases_upload + b200zk_bases_precompute, once per process -- the
 * OnceLock setup of sp1.rs:30,93-95):
 *     quotient  3 iNTT + 3 coset NTT + (a*b - c)/Z_H + 1 coset iNTT    (coset generator 5, the context's NTT root)
 *     commit    [A]1, [B]1, [B]2 over the witness, [L]1 over its private part, [H]1 over the quotient's coefficients
 *     assemble  proof = A (64) | B2 (128, x_im|x_re|y_im|y_re) | C (64), C = [L]1 + [H]1; no blinding (r = s = 0)
 *               and no alpha / beta terms (a key that folds them into variable 0); b200zk_groth16_prove below is the
 *               blinded proof over the ark / gnark key layout
 * Columns: 0 = A_g1, 1 = B_g1 (handle 0 = absent), 2 = B_g2, 3 = L_g1, 4 = H_g1.  count[k] = points of column k this
 * context multiplies; offset[k] = index of the scalar its first point multiplies -- into the witness for columns 0..3
 * (L_g1 of a whole key: offset = number of public inputs incl. the leading 1), into the quotient's coefficients for
 * column 4 (count <= 2^log_n - 1 for a whole key).  A single GPU holds whole columns (offsets 0,0,0,n_public,0); a
 * point-split rank holds a slice of each and passes the slice's start.  Columns that multiply the same scalar slice
 * under the same window plan share ONE digit sort. */
typedef struct b200zk_groth16_pk {
  uint32_t log_n;      /* quotient domain 2^log_n */
  uint32_t reserved;   /* 0 */
  uint64_t handle[5];
  uint64_t count[5];
  uint64_t offset[5];
} b200zk_groth16_pk;
/* witness: scalars (canonical LE unless B200ZK_SCALARS_BE / _MONT), at least max(offset+count) over columns 0..3;
 * a_evals, b_evals, c_evals: (A z), (B z), (C z) on the domain, 2^log_n Montgomery LE elements each.  HOST buffers by
 * default (copied in, left untouched); with B200ZK_G16_INPUTS_DEVICE device pointers, used in place (a_evals is
 * overwritten with the quotient's coefficients, b/c with their coset evaluations).  proof: 256 bytes out;
 * b_g1 (may be NULL): [B]1 as 64 bytes.  One stream, one synchronisation at the end. */
int b200zk_groth16_commit(b200zk_ctx* ctx, const b200zk_groth16_pk* pk, const void* witness, void* a_evals, void* b_evals,
                          void* c_evals, uint32_t flags, void* stream, uint8_t proof[256], uint8_t b_g1[64]);
/* multi-GPU halves: every rank leaves its five partial sums (768 B: A | B1 | B2 | L | H, XYZZ native limbs) in device
 * memory without synchronising; the host side all-gathers the blocks ONCE and every rank folds `count` of them */
int b200zk_groth16_commit_partial(b200zk_ctx* ctx, const b200zk_groth16_pk* pk, const void* witness, void* a_evals,
                                  void* b_evals, void* c_evals, uint32_t flags, void* stream, void* d_partials768);
int b200zk_groth16_fold(b200zk_ctx* ctx, const void* d_partials, size_t count, void* stream, uint8_t proof[256],
                        uint8_t b_g1[64]);

/* ---- zero-knowledge Groth16: the key's alpha / beta / delta terms and the blinding scalars r, s ----------------------
 * The proof ark-groth16 0.5 (create_proof_with_reduction, behind risc0-groth16) and gnark groth16.Prove (behind SP1's
 * wrap) return for the same r and s, over a key in their layout, where alpha and beta are NOT folded into the columns:
 *     A  = alpha1 + sum z_i A_i + r delta1           B2 = beta2 + sum z_i B2_i + s delta2
 *     C  = [L]1 + [H]1 + s A + r B1 - (r s) delta1,   B1 = beta1 + sum z_i B1_i + s delta1
 *     proof = A (64) | B2 (128, x_im|x_re|y_im|y_re) | C (64), EIP-196/197 bytes
 * The key terms are uploaded once with b200zk_g1_bases_upload / b200zk_g2_bases_upload (validated like any column) and
 * must stay plain bases (not precomputed).  r and s are inputs -- the library never draws randomness, so a proof is
 * reproducible -- and must be canonical little-endian values below the group order: a larger value is refused with
 * B200ZK_ERR_NOT_IN_FIELD, not reduced (reducing would bias raw random bytes).  r = s = 0 gives the unblinded proof.
 * B200ZK_ERR_INVALID_ARG: a NULL zk; a term handle that is unknown, of the wrong group or point count, BLS12-381 or
 * precomputed; and in b200zk_groth16_prove, r != 0 with the B_g1 column absent (C needs [B]1). */
typedef struct b200zk_groth16_zk {
  uint64_t g1_terms;  /* resident G1 handle of exactly 3 points: alpha, beta, delta (plain bases, not precomputed) */
  uint64_t g2_terms;  /* resident G2 handle of exactly 2 points: beta, delta */
  uint8_t r[32];      /* canonical little-endian, < group order */
  uint8_t s[32];
} b200zk_groth16_zk;
/* b200zk_groth16_commit_partial followed by b200zk_groth16_fold_zk on one stream, one synchronisation at the end;
 * arguments as b200zk_groth16_commit */
int b200zk_groth16_prove(b200zk_ctx* ctx, const b200zk_groth16_pk* pk, const b200zk_groth16_zk* zk, const void* witness,
                         void* a_evals, void* b_evals, void* c_evals, uint32_t flags, void* stream, uint8_t proof[256]);
/* folds `count` 768-byte blocks of b200zk_groth16_commit_partial (one per rank), then adds the key terms and the
 * blinding once: every rank of a point-split prove folds the all-gathered blocks with the same r and s */
int b200zk_groth16_fold_zk(b200zk_ctx* ctx, const b200zk_groth16_zk* zk, const void* d_partials, size_t count,
                           void* stream, uint8_t proof[256]);

/* ---- BLS12-381 G1 / EIP-4844 blob commitments (SURVEY.md section 8(f) rank 3) -------------------------------------
 * The L2 committer's "commit" step: /root/reference/crates/common/crypto/kzg.rs:259-272 (blob_to_kzg_commitment_and_proof ->
 * c_kzg blob_to_kzg_commitment), /root/reference/crates/common/types/blobs_bundle.rs:90-118, crates/l2/sequencer/
 * l1_committer.rs:1488-1521.  The same Pippenger kernels, instantiated over the 381-bit base field (12 x 32-bit limbs).
 * Points: 48-byte compressed (B200ZK_POINTS_COMPRESSED; bit 7 of byte 0 = compressed, bit 6 = infinity, bit 5 = the larger
 * y) -- the form the trusted setup ships in -- or 96-byte uncompressed big-endian x | y.  Statuses: 2 = a coordinate or a
 * scalar out of its field, 3 = not a curve point / malformed flag bits.  The subgroup check is the trusted setup's
 * business (c-kzg validates it when loading), not repeated here.  The handle works with b200zk_bases_precompute /
 * b200zk_bases_free like any other.  Scalars: 32-byte integers < the BLS12-381 group order r, little-endian limbs or
 * big-endian with B200ZK_SCALARS_BE; either order is checked against r (status 2 otherwise); result: 48 bytes compressed. */
int b200zk_bls12_381_g1_bases_upload(b200zk_ctx* ctx, const void* points, size_t n, uint32_t flags, uint64_t* handle);
int b200zk_bls12_381_g1_msm_resident(b200zk_ctx* ctx, uint64_t handle, const void* scalars, size_t n, uint32_t flags,
                                     uint8_t out[48]);
/* blob_to_kzg_commitment for n_blobs blobs: blob = 4096 x 32-byte big-endian field elements (each < r, else status 2);
 * setup_handle = the 4096 Lagrange-form G1 points of the trusted setup (g1_lagrange_brp order, as c-kzg holds them);
 * commitments: n_blobs x 48 bytes */
int b200zk_kzg_blob_to_commitment(b200zk_ctx* ctx, uint64_t setup_handle, const uint8_t* blobs, size_t n_blobs,
                                  uint8_t* commitments);
/* EIP-4844 proofs, computed on the device: y = p(z) by the barycentric formula, the quotient (p(X) - y) / (X - z) in
 * evaluation form (the spec's special case when z is one of the 4096 roots of unity), and its commitment.  Rules of both:
 *   - setup_handle must be a BLS12-381 handle of exactly 4096 points, else status 4; null pointers with n_blobs > 0: 4;
 *   - every blob element and every z must be < r.  All are checked before any MSM; a failure returns 2, writes no output,
 *     and b200zk_last_error names the blob;
 *   - n_blobs = 0 returns 0;
 *   - an identity commitment or proof is encoded as 0xc0 | 0..0 and the status is still 0.
 * blob_to_kzg_commitment_and_proof (/root/reference/crates/common/crypto/kzg.rs:259-272) for n_blobs blobs: the commitment,
 * then the proof at the Fiat-Shamir challenge z = hash_to_bls_field(SHA-256("FSBLOBVERIFY_V1_" | 4096 as 16-byte big-endian
 * | blob | commitment)).  The commitments are read back once for the hash (on the host), then the proofs are computed.
 * commitments and proofs: n_blobs x 48 bytes compressed each. */
int b200zk_kzg_blob_to_commitment_and_proof(b200zk_ctx* ctx, uint64_t setup_handle, const uint8_t* blobs, size_t n_blobs,
                                            uint8_t* commitments, uint8_t* proofs);
/* c-kzg compute_kzg_proof for n_blobs (blob, z) pairs: z and y are n_blobs x 32-byte big-endian; proofs n_blobs x 48 bytes */
int b200zk_kzg_compute_proof(b200zk_ctx* ctx, uint64_t setup_handle, const uint8_t* blobs, size_t n_blobs,
                             const uint8_t* z, uint8_t* proofs, uint8_t* y);

/* ---- the BLS12-381 pairing and EIP-4844 KZG verification ----------------------------------------------------------
 * The three reference calls that rest on a BLS12-381 pairing:
 *   bls12_381_pairing_check   Crypto::bls12_381_pairing_check (EIP-2537 pairing precompile 0x0f), provider.rs:642-672
 *   kzg_verify_proof          Crypto::verify_kzg_proof (POINT_EVALUATION precompile 0x0a), provider.rs:463-507
 *   kzg_verify_blob_proof     Crypto::verify_blob_kzg_proof / kzg::verify_kzg_proof_batch (blob transactions),
 *                             provider.rs:509-544, crates/common/crypto/kzg.rs:168-192
 * The pairing is the optimal ate pairing with line coefficients prepared per G2 point; a check asks whether a product of
 * pairings is one.
 *
 * G2 bases: n points in the 96-byte compressed ZCash form (the trusted setup's g2_monomial): x.c1 | x.c0 big-endian, flag
 * bits in byte 0 (bit 7 compressed, bit 6 infinity, bit 5 the larger y: y.c1 > (p-1)/2, or y.c1 = 0 and y.c0 > (p-1)/2).
 * B200ZK_POINTS_COMPRESSED is required (status 4 otherwise).  Status 2: x.c0 or x.c1 >= p; 3: bad flag bits, not on the
 * twist y^2 = x^3 + 4(1 + u), or not in the order-r subgroup (checked here, unlike G1 bases: a non-subgroup [tau]2 would
 * make the verifier unsound).  The handle is freed by b200zk_bases_free; every MSM entry point, b200zk_bases_precompute
 * and the BLS12-381 G1 / KZG prove calls refuse it with status 4. */
int b200zk_bls12_381_g2_bases_upload(b200zk_ctx* ctx, const void* points, size_t n, uint32_t flags, uint64_t* handle);
/* The EIP-2537 pairing check, `count` checks per call.  Check i covers pairs [pair_offsets[i], pair_offsets[i+1]) of
 * `pairs`, 384 bytes each: G1 (128 B, x | y) then G2 (256 B, x.c0 | x.c1 | y.c0 | y.c1); every Fp is 64 bytes, 16 zero
 * bytes then 48 bytes big-endian; all-zero is the identity.  Per check: status[i] = 2 when a coordinate is >= p or a
 * padding byte is nonzero (checked for every point of the check before any curve check), 3 when a point is not on its
 * curve or not in the order-r subgroup (G1 and G2 both); result[i] = 1 when the product of its pairings is one (an empty
 * check, and pairs with an identity side, contribute 1), 0 otherwise or when status[i] != 0. */
int b200zk_bls12_381_pairing_check_batch(b200zk_ctx* ctx, const uint8_t* pairs /* 384 B each */, const uint32_t* pair_offsets /* count+1 */,
                                         size_t count, uint8_t* result /* count */, uint8_t* status /* count */);
/* KZG verification against a G2 setup handle: a BLS12-381 G2 handle of at least 2 points whose point 0 is the G2 generator;
 * point 1 is [tau]2.  Anything else returns 4.
 * c-kzg verify_kzg_proof for n independent items: commitment and proof 48-byte compressed G1, z and y 32-byte big-endian.
 * Per item: status[i] = 2 when z or y >= r or a coordinate >= p, 3 when a commitment or proof has bad flag bits, is off the
 * curve or not in the order-r subgroup (c-kzg validate_kzg_g1; the identity is valid); result[i] = 1 when the proof is
 * valid.  A failed item reports 0 and does not affect the others. */
int b200zk_kzg_verify_proof_batch(b200zk_ctx* ctx, uint64_t g2_setup, const uint8_t* commitments /* 48 n */, const uint8_t* z /* 32 n */,
                                  const uint8_t* y /* 32 n */, const uint8_t* proofs /* 48 n */, size_t n, uint8_t* result /* n */,
                                  uint8_t* status /* n */);
/* c-kzg verify_blob_kzg_proof_batch: one answer for n (blob, commitment, proof) triples, *valid = 1 or 0.  Bad input is an
 * error, not 0: a blob element >= r returns 2, a malformed or non-subgroup commitment or proof 2 or 3 as above; then
 * *valid is not written and b200zk_last_error names the blob.  n = 0 returns 0 with *valid = 1. */
int b200zk_kzg_verify_blob_proof_batch(b200zk_ctx* ctx, uint64_t g2_setup, const uint8_t* blobs, const uint8_t* commitments,
                                       const uint8_t* proofs, size_t n, int* valid);

/* ---- EIP-7594 cells (PeerDAS, blob bundles of wrapper version 1) ---------------------------------------------------
 *   kzg_compute_cells             c-kzg compute_cells, crates/common/crypto/kzg.rs:89-91
 *   kzg_verify_cell_proof_batch   kzg::verify_cell_kzg_proof_batch, kzg.rs:72-113, reached from BlobsBundle::verify_kzg_proofs
 *                                 (crates/common/types/blobs_bundle.rs:152-173) for every post-Osaka blob transaction
 *   kzg_blob_to_commitment_and_cell_proofs
 *                                 kzg::blob_to_commitment_and_cell_proofs (c-kzg compute_cells_and_kzg_proofs), kzg.rs:275-293,
 *                                 called per blob by BlobsBundle::create_from_blobs for wrapper version 1 (blobs_bundle.rs:101-110)
 * A blob (4096 x 32-byte big-endian elements, each < r, else status 2 with b200zk_last_error naming the blob) lists p's
 * values on the 4096 roots of unity in bit-reversed order, root 7^((r-1)/4096).  Its extension lists p on the 8192
 * roots of unity in bit-reversed order, split into CELLS_PER_EXT_BLOB = 128 cells of FIELD_ELEMENTS_PER_CELL = 64
 * elements (2048 bytes); cells 0..63 are the blob itself.
 * kzg_compute_cells: cells = n_blobs x 128 x 2048 bytes.  n_blobs = 0 returns 0; null pointers with n_blobs > 0: 4. */
int b200zk_kzg_compute_cells(b200zk_ctx* ctx, const uint8_t* blobs, size_t n_blobs, uint8_t* cells /* n_blobs x 128 x 2048 B */);
/* The commitment and the 128 cell proofs of each of n_blobs blobs, by FK20.  Cell k's proof is [q_k(tau)]1 with
 * q_k = (p - I_k) / (X^64 - h_k^64), I_k = p mod (X^64 - h_k^64), h_k = w_8192^brp7(k) the first root of the cell's coset.
 * g1_lagrange: the 4096-point Lagrange-form G1 handle of the KZG calls above (the commitment is an MSM over it).
 * g1_monomial: a 4096-point BLS12-381 G1 handle (b200zk_bls12_381_g1_bases_upload) holding the setup's g1_monomial points
 * [tau^i]1 in order; that both handles describe one tau is the setup's business.  The FK20 table derived from it (64 x 128
 * points, 0.8 MB) is built on the handle's first call here, kept with the handle and freed by b200zk_bases_free.
 * Rules: a G2 handle, an unknown handle or one of the wrong size returns 4, as do null pointers with n_blobs > 0;
 * n_blobs = 0 returns 0; every blob element is checked < r before any MSM, and a failure returns 2, writes nothing and
 * names the blob and element in b200zk_last_error; an identity commitment or proof is 0xc0 | 0..0 with status 0.
 * commitments: n_blobs x 48 bytes; proofs: n_blobs x 128 x 48 bytes, blob-major with the cell index inner (compressed G1). */
int b200zk_kzg_blob_to_commitment_and_cell_proofs(b200zk_ctx* ctx, uint64_t g1_lagrange, uint64_t g1_monomial, const uint8_t* blobs,
                                                  size_t n_blobs, uint8_t* commitments /* 48 n */, uint8_t* proofs /* 128 x 48 n */);
/* verify_cell_kzg_proof_batch over whole blobs, the shape the reference calls it with: every blob's 128 cells, cell
 * indices 0..127, each commitment standing for its blob's 128 cells; proofs are blob-major, 128 per blob, cell index inner
 * (48-byte compressed G1 each).  One answer, *valid = 1 or 0, from one two-pairing check of the universal equation
 *   e(sum r^k pi_k, [tau^64]2) = e(sum_i (sum_(k in blob i) r^k) C_i - [sum r^k I_k(tau)]1 + sum r^k h_k^64 pi_k, [1]2)
 * with I_k the interpolation polynomial of cell k on its coset h_k <w_64> and r the Fiat-Shamir challenge: SHA-256 of
 * "RCKZGCBATCH__V1_", the sizes (4096, 64, n_blobs, 128 n_blobs as u64 big-endian), the commitments, then per cell its
 * blob and cell index (u64 big-endian), its 64 elements and its proof, reduced mod r (the spec's construction; the
 * commitments are not deduplicated, so r need not equal c-kzg's byte for byte).
 * g1_setup: the 4096-point Lagrange-form G1 handle of the KZG calls above ([sum r^k I_k(tau)]1 is an MSM over it).
 * g2_setup: a BLS12-381 G2 handle of at least 65 points whose point 0 is the G2 generator; point 64 is [tau^64]2 (c-kzg's
 * setup ships 65 g2_monomial points for this).  Anything else returns 4.
 * Bad input is an error and *valid is not written: a blob element >= r returns 2; a commitment or proof with a coordinate
 * >= p returns 2; bad flag bits, a point off the curve or outside the order-r subgroup returns 3 (the identity is valid);
 * b200zk_last_error names the blob (and cell).  Null pointers with n_blobs > 0 return 4.  n_blobs = 0 returns 0 with
 * *valid = 1. */
int b200zk_kzg_verify_cell_proof_batch(b200zk_ctx* ctx, uint64_t g1_setup, uint64_t g2_setup, const uint8_t* blobs,
                                       const uint8_t* commitments /* 48 n */, const uint8_t* proofs /* 128 x 48 n */, size_t n_blobs,
                                       int* valid);

/* ---- EIP-2537 G1/G2 addition and multi-scalar multiplication -------------------------------------------------------
 * The Prague precompiles 0x0b-0x0e, `count` independent items per call, HOST buffers:
 *   bls12_381_g1_add  Crypto::bls12_381_g1_add, provider.rs:549-562 (levm BLS12_G1ADD, precompiles.rs:1056-1107)
 *   bls12_381_g1_msm  Crypto::bls12_381_g1_msm, provider.rs:566-593 (levm BLS12_G1MSM, precompiles.rs:1109-1165)
 *   bls12_381_g2_add  Crypto::bls12_381_g2_add, provider.rs:596-609 (levm BLS12_G2ADD, precompiles.rs:1167-1244)
 *   bls12_381_g2_msm  Crypto::bls12_381_g2_msm, provider.rs:613-640 (levm BLS12_G2MSM, precompiles.rs:1246-1315)
 * Encodings as the pairing check: every Fp is 64 bytes, 16 zero bytes then 48 bytes big-endian; G1 = x | y (128 B), G2 =
 * x.c0 | x.c1 | y.c0 | y.c1 (256 B); all-zero is the identity.  An MSM pair is a point followed by a 32-byte big-endian
 * scalar (G1 160 B, G2 288 B); MSM call i covers pairs [pair_offsets[i], pair_offsets[i+1]).
 * The return value reports infrastructure errors only; input errors are per item in status[i], with the table of the
 * BN254 batches (the provider's parse_bls12_g1 / _g2 / _scalar, provider.rs:724-795):
 *   0 ok, 1 ok and the result is the identity,
 *   2 a coordinate >= p or a nonzero padding byte (checked for every point of the item before any curve check, so 2
 *     outranks 3 within an item),
 *   3 a point is off its curve; for the MSM calls also a point outside the order-r subgroup.
 * Addition checks no subgroup (EIP-2537 and the provider ask only for the curve).  The MSM checks every non-identity point,
 * including those whose scalar is zero (the provider's is_torsion_free).  Scalars are any 256-bit value: k P = (k mod r) P
 * for a subgroup point, so a scalar >= r is not an error.  An empty MSM call returns the identity with status 1, as the
 * provider does (levm refuses empty calldata before it).  out[i] is the precompile's own output (padded EIP-2537, the
 * identity all zero); a failed item's output is all zero.  count = 0 returns 0; null pointers, pair_offsets[0] != 0 or
 * decreasing offsets return 4 with b200zk_last_error set. */
int b200zk_bls12_381_g1_add_batch(b200zk_ctx* ctx, const uint8_t* a /* count*128 */, const uint8_t* b /* count*128 */, size_t count,
                                  uint8_t* out /* count*128 */, uint8_t* status /* count */);
int b200zk_bls12_381_g2_add_batch(b200zk_ctx* ctx, const uint8_t* a /* count*256 */, const uint8_t* b /* count*256 */, size_t count,
                                  uint8_t* out /* count*256 */, uint8_t* status /* count */);
int b200zk_bls12_381_g1_msm_batch(b200zk_ctx* ctx, const uint8_t* pairs /* 160 B each */, const uint32_t* pair_offsets /* count+1 */,
                                  size_t count, uint8_t* out /* count*128 */, uint8_t* status /* count */);
int b200zk_bls12_381_g2_msm_batch(b200zk_ctx* ctx, const uint8_t* pairs /* 288 B each */, const uint32_t* pair_offsets /* count+1 */,
                                  size_t count, uint8_t* out /* count*256 */, uint8_t* status /* count */);

/* ---- secp256k1 signer recovery (ECRECOVER) -------------------------------------------------------------------------
 * `count` independent items per call, HOST buffers:
 *   secp256k1_ecrecover  Crypto::secp256k1_ecrecover, provider.rs:63-88 (levm ECRECOVER 0x01, precompiles.rs:456-510)
 *   recover_signer       Crypto::recover_signer, provider.rs:153-171 (transaction senders, EIP-7702 authorities): pass
 *                        B200ZK_ECRECOVER_LOW_S and take the address from bytes 12..32 of out[i]
 * Item i: sigs[65 i ..] = r (32 B big-endian) | s (32 B big-endian) | recid (1 B), msgs[32 i ..] = the 32-byte message
 * hash.  out[32 i ..] = keccak256(X | Y) of the recovered public key (X, Y 32-byte big-endian).  The checks run in this
 * order and the first failure sets status[i] (a failed item's output is all zero):
 *   2 InvalidSignature    with B200ZK_ECRECOVER_LOW_S: s > n/2 (EIP-2)
 *   4 InvalidRecoveryId   recid > 3
 *   2 InvalidSignature    r >= n or s >= n
 *   3 RecoveryFailed      r = 0 or s = 0; recid 2 or 3 with r >= p - n (otherwise x = r + n); no curve point has
 *                         abscissa x (x^3 + 7 is not a square); Q = r^-1 (s R - z G) is the identity
 *   0 ok
 * R is the point with abscissa x and y parity recid & 1, z the hash as a 256-bit integer reduced mod n.  This is the
 * libsecp256k1 path, the reference's default build; its k256 fallback (provider.rs:90-151) rejects recids 2 and 3.  Real
 * callers pass 0 or 1 (the precompile maps v = 27 / 28, transactions carry a y-parity bit).
 * count = 0 returns 0; null pointers or unknown flag bits return 4 with b200zk_last_error set.  The table of G multiples
 * the call reads is built on the device on the context's first call (256 KB, kept until b200zk_destroy). */
#define B200ZK_ECRECOVER_LOW_S 1u /* reject s > n/2 with status 2 (EIP-2, Crypto::recover_signer) */
int b200zk_secp256k1_ecrecover_batch(b200zk_ctx* ctx, const uint8_t* sigs /* count*65 */, const uint8_t* msgs /* count*32 */,
                                     size_t count, uint32_t flags, uint8_t* out /* count*32 */, uint8_t* status /* count */);

/* ---- secp256r1 (P-256) signature verification (P256VERIFY) ---------------------------------------------------------
 * `count` independent items per call, HOST buffers:
 *   secp256r1_verify  Crypto::secp256r1_verify, provider.rs:415-459 (levm P256VERIFY 0x0100, precompiles.rs:987-1043,
 *                     EIP-7951; on every L2 and on L1 from Osaka)
 * Item i: inputs[160 i ..] = the precompile's calldata h | r | s | qx | qy, five 32-byte big-endian words (the message
 * hash, the signature, the public key).  result[i] = 1 when the signature verifies, 0 otherwise; as in the trait there is
 * no per-item status.  The rules, in order (p256 0.13.2's verify_prehash as the provider calls it, and EIP-7951):
 *   0  r or s outside [1, n - 1] (provider.rs:432-434)
 *   0  qx >= p or qy >= p (non-canonical encodings are rejected, never reduced)
 *   0  (qx, qy) not on y^2 = x^3 - 3x + b, (0, 0) included; the cofactor is 1, so there is no subgroup check
 *   0  R' = (z s^-1) G + (r s^-1) Q is the identity, z = h mod n (the hash as a 256-bit integer)
 *   1  iff x(R') mod n = r
 * High s is accepted: (r, s) and (r, n - s) both verify.  The 160-byte length check and the gas stay with the caller.
 * count = 0 returns 0; null pointers return 4 with b200zk_last_error set.  The table of G multiples the call reads is
 * built on the device on the context's first call (256 KB, kept until b200zk_destroy). */
int b200zk_secp256r1_verify_batch(b200zk_ctx* ctx, const uint8_t* inputs /* count*160 */, size_t count, uint8_t* result /* count */);

/* ---- batched EIP-196 / EIP-197 precompile arithmetic (SURVEY.md section 8(f) rank 4) ------------------------------
 * The three BN254 calls of the reference's `Crypto` trait, `count` independent items per call, HOST buffers:
 *   bn254_g1_add         crates/common/crypto/provider.rs:201-234   (levm ecadd,     crates/vm/levm/src/precompiles.rs:692-716)
 *   bn254_g1_mul         crates/common/crypto/provider.rs:239-272   (levm ecmul,     precompiles.rs:719-745)
 *   bn254_pairing_check  crates/common/crypto/provider.rs:277-330   (levm ecpairing, precompiles.rs:821-860)
 * Encodings: G1 = 64 B big-endian x|y, (0,0) = identity; G2 = 128 B x_im|x_re|y_im|y_re; scalars 32 B big-endian
 * (any 256-bit value: the group has prime order).  The function's return value reports infrastructure errors only;
 * input errors are PER ITEM in status[i], with the ZisK-style table (crates/guest-program/src/crypto/zisk.rs:144-172):
 *   0 ok, 1 ok and the result is the identity, 2 a coordinate >= p (levm: CoordinateExceedsFieldModulus,
 *   checked for every point of the item before any curve check), 3 a point is not on the curve or (G2) not in the
 *   order-r subgroup.  Outputs of failed items are zero.
 * The reference's own vectors for this surface (14 ecpairing cases + the out-of-range case,
 * test/tests/levm/precompile_tests.rs:17-151; 7*(1,2) of test/tests/l2/integration_tests.rs:572) run through these
 * entry points in tests/test_gpu_parity.py. */
int b200zk_bn254_g1_add_batch(b200zk_ctx* ctx, const uint8_t* a /* count*64 */, const uint8_t* b /* count*64 */, size_t count,
                              uint8_t* out /* count*64 */, uint8_t* status /* count */);
int b200zk_bn254_g1_mul_batch(b200zk_ctx* ctx, const uint8_t* points /* count*64 */, const uint8_t* scalars /* count*32 */, size_t count,
                              uint8_t* out /* count*64 */, uint8_t* status /* count */);
/* check i covers pairs [pair_offsets[i], pair_offsets[i+1]) of `pairs` (192 B each: G1 | G2); result[i] = 1 when
 * the product of its pairings is one (an empty check is 1), 0 otherwise or when status[i] != 0 */
int b200zk_bn254_pairing_check_batch(b200zk_ctx* ctx, const uint8_t* pairs, const uint32_t* pair_offsets /* count+1 */, size_t count,
                                     uint8_t* result /* count */, uint8_t* status /* count */);

#ifdef __cplusplus
}
#endif
#endif /* B200ZK_H */
