// groth16.cu -- the Groth16 prove arithmetic as ONE call of the C ABI (SURVEY.md section 8b "b200zk_groth16_commit",
// section 8f row 1): what the SNARK wrap behind ProofFormat::Groth16 computes after witness generation
// (/root/reference/crates/prover/src/backend/sp1.rs:97-134 -> gnark `groth16.Prove`; risc0.rs:24-29,71-82 ->
// risc0-groth16), over a proving key that already lives in HBM:
//
//   quotient   3 iNTT (A.z, B.z, C.z on the domain -> coefficients), 3 coset NTT, (a*b - c)/Z_H pointwise, 1 coset iNTT
//   commit     [A]1 = <pk.A_g1, z>   [B]1 = <pk.B_g1, z>   [B]2 = <pk.B_g2, z>   [L]1 = <pk.L_g1, z_private>   [H]1 = <pk.H_g1, h>
//   assemble   proof = A | B2 | C,  C = [L]1 + [H]1         (EIP-196/197 bytes, 256 B; no blinding: r = s = 0)
//   or, b200zk_groth16_prove / _fold_zk: the ark-groth16 / gnark proof with the key's alpha / beta / delta terms and the
//              caller's blinding scalars r, s (groth16_assemble_zk in msm.cu)
//
// Everything is enqueued on one stream with no host round trip in between; columns that multiply the same scalar
// slice share ONE digit sort (msm_run sort_mode 1/2), and the five results stay on the device as XYZZ partial sums
// (768 B: A | B1 | B2 | L | H) so that the multi-GPU driver can all-gather them ONCE and fold
// (b200zk_groth16_commit_partial + b200zk_groth16_fold).
#include "common.cuh"
#include <cstring>

namespace b200zk {

static int stage(b200zk_ctx* ctx, DevBuf& buf, const void* host, size_t bytes, cudaStream_t st, void** out) {
  B2_TRY(ensure(ctx, buf, bytes + 32));
  if (bytes) B2_CUDA(ctx, cudaMemcpyAsync(buf.p, host, bytes, cudaMemcpyHostToDevice, st));
  *out = buf.p;
  return B200ZK_OK;
}

int groth16_commit_partials(b200zk_ctx* ctx, const b200zk_groth16_pk* pk, const void* witness, void* a_evals, void* b_evals, void* c_evals,
                            uint32_t flags, cudaStream_t st, void* d_partials) {
  NvtxRange nvtx_g16("b200zk:groth16_commit");
  if (!pk || !d_partials) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_commit: null argument");
  if (pk->log_n > 28) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_commit: log_n > 28");
  const size_t n = (size_t)1 << pk->log_n;
  const bool on_device = flags & B200ZK_G16_INPUTS_DEVICE, h_ready = flags & B200ZK_G16_H_COEFFS;
  const BasesEntry* col[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
  size_t wit_end = 0;  // witness entries the columns reach
  for (int k = 0; k < 5; ++k) {
    if (!pk->handle[k]) { if (k == 1) continue; return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_commit: only the B_g1 column may be absent"); }
    col[k] = find_bases(ctx, pk->handle[k], k == 2 ? Group::Bn254G2 : Group::Bn254G1, "groth16_commit: unknown handle or wrong group for a column");
    if (!col[k]) return B200ZK_ERR_INVALID_ARG;
    if (pk->count[k] > col[k]->n) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_commit: a column count exceeds its resident bases");
    if (k < 4 && pk->offset[k] + pk->count[k] > wit_end) wit_end = pk->offset[k] + pk->count[k];
  }
  if (pk->offset[4] + pk->count[4] > n) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_commit: the H column reaches past the quotient's 2^log_n coefficients");
  if ((!witness && wit_end) || !a_evals || (!h_ready && (!b_evals || !c_evals))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_commit: null argument");

  // ---- inputs into HBM (host buffers are staged; device buffers are used in place and a_evals is overwritten with H)
  const uint8_t* d_wit = (const uint8_t*)witness;
  void *d_a = a_evals, *d_b = b_evals, *d_c = c_evals;
  if (!on_device) {
    void* p;
    B2_TRY(stage(ctx, ctx->ws_scalars, witness, wit_end * 32, st, &p)); d_wit = (const uint8_t*)p;
    B2_TRY(stage(ctx, ctx->ws_g16[0], a_evals, n * 32, st, &d_a));
    if (!h_ready) { B2_TRY(stage(ctx, ctx->ws_g16[1], b_evals, n * 32, st, &d_b)); B2_TRY(stage(ctx, ctx->ws_g16[2], c_evals, n * 32, st, &d_c)); }
  }
  // ---- quotient: H(x) = (A(x) B(x) - C(x)) / Z_H(x), coefficients left in d_a (Montgomery)
  if (!h_ready) {
    NvtxRange nvtx_q("b200zk:groth16_quotient");
    void* polys[3] = {d_a, d_b, d_c};
    for (void* p : polys) {
      B2_TRY(ntt_run(ctx, p, pk->log_n, B200ZK_NTT_INVERSE, nullptr, st));
      B2_TRY(ntt_run(ctx, p, pk->log_n, B200ZK_NTT_COSET, nullptr, st));
    }
    const uint32_t* d_zinv = nullptr;
    B2_TRY(fr_coset_zinv_dev(ctx, pk->log_n, st, &d_zinv));
    B2_TRY(fr_quotient_dev(ctx, d_a, d_b, d_c, d_a, n, d_zinv, st));
    B2_TRY(ntt_run(ctx, d_a, pk->log_n, B200ZK_NTT_INVERSE | B200ZK_NTT_COSET, nullptr, st));
  }
  // ---- the five MSMs; columns over the same scalar slice with the same plan share one sort
  static const size_t kPartialOff[5] = {0, 128, 256, 512, 640};
  uint8_t* out = (uint8_t*)d_partials;
  const uint32_t wflags = flags & (B200ZK_SCALARS_BE | B200ZK_SCALARS_MONT);
  int prev = -1;  // previous witness column that ran (candidate sort donor)
  for (int k = 0; k < 4; ++k) {
    if (!col[k]) { B2_CUDA(ctx, cudaMemsetAsync(out + kPartialOff[k], 0, 128, st)); continue; }  // absent B_g1: identity (ZZ = 0)
    const size_t cnt = pk->count[k];
    const uint8_t* sc = d_wit + pk->offset[k] * 32;
    bool share = prev >= 0 && cnt >= 2 && pk->offset[prev] == pk->offset[k] && pk->count[prev] == cnt && col[prev]->table_c == col[k]->table_c &&
                 (!col[k]->table_c || col[prev]->n == col[k]->n);
    // is this column followed by one that can reuse its sort?  (then it must run as one chunk and keep it)
    bool donor = false;
    for (int j = k + 1; j < 4 && !donor; ++j)
      donor = col[j] && cnt >= 2 && pk->offset[j] == pk->offset[k] && pk->count[j] == cnt && col[j]->table_c == col[k]->table_c && (!col[k]->table_c || col[j]->n == col[k]->n);
    const int mode = share ? 2 : (donor ? 1 : 0);
    int rc = (k == 2) ? msm_run_g2(ctx, col[k]->d.p, sc, cnt, wflags, st, out + kPartialOff[k], col[k]->table_c, col[k]->n, nullptr, mode)
                      : msm_run_g1(ctx, col[k]->d.p, sc, cnt, wflags, st, out + kPartialOff[k], col[k]->table_c, col[k]->n, nullptr, mode);
    if (rc > B200ZK_OK_INFINITY) return rc;
    if (!share) prev = k;
  }
  {
    const uint8_t* hc = (const uint8_t*)d_a + pk->offset[4] * 32;
    int rc = msm_run_g1(ctx, col[4]->d.p, hc, pk->count[4], B200ZK_SCALARS_MONT, st, out + kPartialOff[4], col[4]->table_c, col[4]->n, nullptr, 0);
    if (rc > B200ZK_OK_INFINITY) return rc;
  }
  return B200ZK_OK;
}

// x (32 bytes little-endian) < the group order r: blinding scalars are refused, not reduced, so that raw random bytes
// cannot skew their distribution
static bool fr_canonical(const uint8_t* x) {
  for (int i = 7; i >= 0; --i) {
    const uint32_t w = (uint32_t)x[4 * i] | (uint32_t)x[4 * i + 1] << 8 | (uint32_t)x[4 * i + 2] << 16 | (uint32_t)x[4 * i + 3] << 24;
    if (w != FrCfg::mod(i)) return w < FrCfg::mod(i);
  }
  return false;
}

// the key terms of a b200zk_groth16_zk: plain (not precomputed) BN254 bases of the right group and point count
int groth16_zk_terms(b200zk_ctx* ctx, const b200zk_groth16_zk* zk, const void** g1, const void** g2) {
  if (!zk) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16 zk: null argument");
  static const char* kG1 = "groth16 zk: g1_terms must be a plain G1 handle of 3 points (alpha, beta, delta)";
  static const char* kG2 = "groth16 zk: g2_terms must be a plain G2 handle of 2 points (beta, delta)";
  const BasesEntry* e1 = find_bases(ctx, zk->g1_terms, Group::Bn254G1, kG1);
  if (!e1) return B200ZK_ERR_INVALID_ARG;
  if (e1->table_c || e1->n != 3) return fail(ctx, B200ZK_ERR_INVALID_ARG, kG1);
  const BasesEntry* e2 = find_bases(ctx, zk->g2_terms, Group::Bn254G2, kG2);
  if (!e2) return B200ZK_ERR_INVALID_ARG;
  if (e2->table_c || e2->n != 2) return fail(ctx, B200ZK_ERR_INVALID_ARG, kG2);
  if (!fr_canonical(zk->r) || !fr_canonical(zk->s)) return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, "groth16 zk: r or s is not below the group order");
  *g1 = e1->d.p;
  *g2 = e2->d.p;
  return B200ZK_OK;
}

static int fold_zk(b200zk_ctx* ctx, const b200zk_groth16_zk* zk, const void* g1, const void* g2, const void* d_partials, size_t count,
                   cudaStream_t st, uint8_t proof[256]) {
  B2_TRY(ensure(ctx, ctx->ws_out, 512));
  B2_TRY(groth16_assemble_zk_dev(ctx, d_partials, count, g1, g2, zk->r, zk->s, st, ctx->ws_out.p));
  B2_CUDA(ctx, cudaMemcpyAsync(ctx->h_pinned, ctx->ws_out.p, 256, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  memcpy(proof, ctx->h_pinned, 256);
  return B200ZK_OK;
}

}  // namespace b200zk

using namespace b200zk;

extern "C" {

int b200zk_groth16_commit_partial(b200zk_ctx* ctx, const b200zk_groth16_pk* pk, const void* witness, void* a_evals, void* b_evals, void* c_evals,
                                  uint32_t flags, void* stream, void* d_partials768) {
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  DeviceGuard guard(ctx);
  return groth16_commit_partials(ctx, pk, witness, a_evals, b_evals, c_evals, flags, pick_stream(ctx, stream), d_partials768);
}

int b200zk_groth16_fold(b200zk_ctx* ctx, const void* d_partials, size_t count, void* stream, uint8_t proof[256], uint8_t b_g1[64]) {
  if (!ctx || !proof || (!d_partials && count)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_fold: null argument");
  DeviceGuard guard(ctx);
  cudaStream_t st = pick_stream(ctx, stream);
  B2_TRY(ensure(ctx, ctx->ws_out, 512));
  B2_TRY(groth16_assemble_dev(ctx, d_partials, count, st, ctx->ws_out.p));
  B2_CUDA(ctx, cudaMemcpyAsync(ctx->h_pinned, ctx->ws_out.p, 336, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  memcpy(proof, ctx->h_pinned, 256);
  if (b_g1) memcpy(b_g1, ctx->h_pinned + 256, 64);
  return B200ZK_OK;
}

int b200zk_groth16_commit(b200zk_ctx* ctx, const b200zk_groth16_pk* pk, const void* witness, void* a_evals, void* b_evals, void* c_evals,
                          uint32_t flags, void* stream, uint8_t proof[256], uint8_t b_g1[64]) {
  if (!ctx || !proof) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_commit: null argument");
  DeviceGuard guard(ctx);
  cudaStream_t st = pick_stream(ctx, stream);
  B2_TRY(ensure(ctx, ctx->ws_g16[3], 1024));
  B2_TRY(groth16_commit_partials(ctx, pk, witness, a_evals, b_evals, c_evals, flags, st, ctx->ws_g16[3].p));
  return b200zk_groth16_fold(ctx, ctx->ws_g16[3].p, 1, (void*)st, proof, b_g1);
}

int b200zk_groth16_fold_zk(b200zk_ctx* ctx, const b200zk_groth16_zk* zk, const void* d_partials, size_t count, void* stream, uint8_t proof[256]) {
  if (!ctx || !proof || (!d_partials && count)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_fold_zk: null argument");
  DeviceGuard guard(ctx);
  const void *g1 = nullptr, *g2 = nullptr;
  B2_TRY(groth16_zk_terms(ctx, zk, &g1, &g2));
  return fold_zk(ctx, zk, g1, g2, d_partials, count, pick_stream(ctx, stream), proof);
}

int b200zk_groth16_prove(b200zk_ctx* ctx, const b200zk_groth16_pk* pk, const b200zk_groth16_zk* zk, const void* witness, void* a_evals, void* b_evals,
                         void* c_evals, uint32_t flags, void* stream, uint8_t proof[256]) {
  if (!ctx || !proof || !pk) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_prove: null argument");
  DeviceGuard guard(ctx);
  const void *g1 = nullptr, *g2 = nullptr;
  B2_TRY(groth16_zk_terms(ctx, zk, &g1, &g2));
  bool r_zero = true;
  for (int i = 0; i < 32; ++i) r_zero = r_zero && !zk->r[i];
  // C = ... + r [B]1: only r = 0 may skip the B_g1 column (what ark-groth16 does)
  if (!pk->handle[1] && !r_zero) return fail(ctx, B200ZK_ERR_INVALID_ARG, "groth16_prove: r != 0 needs the B_g1 column");
  cudaStream_t st = pick_stream(ctx, stream);
  B2_TRY(ensure(ctx, ctx->ws_g16[3], 1024));
  B2_TRY(groth16_commit_partials(ctx, pk, witness, a_evals, b_evals, c_evals, flags, st, ctx->ws_g16[3].p));
  return fold_zk(ctx, zk, g1, g2, ctx->ws_g16[3].p, 1, st, proof);
}

}  // extern "C"
