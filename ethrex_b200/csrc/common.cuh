// common.cuh -- context, workspace and launch bookkeeping shared by the translation units of libb200zk.so.
#pragma once
#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h>  // header-only NVTX v3: ranges show up in nsys / ncu --nvtx timelines, no-ops otherwise
#include <cstdint>
#include <cstdio>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "../../include/b200zk.h"
#include "curve.cuh"
#include "bls381.cuh"

namespace b200zk {

template <> struct CurveB<Fp381> {
  static B2_D Fp381 b() { Fp381 four = Fp381::zero(); four.v[0] = 4; return Fp381::to_mont(four); }  // y^2 = x^3 + 4
};

// a device allocation that frees itself: grown by ensure(), move-only
struct DevBuf {
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(DevBuf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  DevBuf& operator=(DevBuf&& o) noexcept {
    if (this != &o) { reset(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
    return *this;
  }
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { reset(); }
  void reset() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

// a table built on first use by once_table(); consumers on other streams wait on `ready`
struct OnceTable {
  DevBuf buf;
  cudaEvent_t ready = nullptr;
  bool built = false;  // set only once the build is enqueued and its event recorded
  OnceTable() = default;
  OnceTable(OnceTable&& o) noexcept : buf(std::move(o.buf)), ready(o.ready), built(o.built) { o.ready = nullptr; o.built = false; }
  ~OnceTable() { if (ready) cudaEventDestroy(ready); }
};

struct TwiddleSet {   // per (log_n, direction): see ntt.cu
  void* d = nullptr;  // device allocation holding all tables
  size_t bytes = 0;
  uint32_t gen[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // coset tables: the generator they were built for
  uint32_t root[8] = {0, 0, 0, 0, 0, 0, 0, 0};  // the 2^28-th root of unity the tables were built for (all zero = default)
  cudaEvent_t ready = nullptr;  // recorded behind the build kernel: consumers on OTHER streams wait on it
};

// the MSM's digit sort (msm.cu sort_digits) and its run offsets: hist / offsets / idx are the sort, run_off numbers the
// accumulation's runs, tsum is scan scratch; digits and cursor serve the one-pass sort only, key / ctab / cnt2 the
// two-level sort only
struct SortWorkspace {
  DevBuf hist, offsets, cursor, run_off, tsum, digits, idx, key, ctab, cnt2;
};

// Bls12G1: Fp381 Montgomery, 96 B affine, the KZG trusted setup; Bls12G2: Fp2 over Fp381, 192 B affine, followed by the
// prepared Miller-loop lines of points 0 and 1
enum class Group { Bn254G1, Bn254G2, Bls12G1, Bls12G2 };

// native affine point bytes and scalar bits (ScalarBits<F>: BLS12-381's group order has one more bit) of a group
struct GroupSizes { size_t point; uint32_t scalar_bits; };
inline GroupSizes group_sizes(Group g) {
  switch (g) {
    case Group::Bn254G1: return {64, 255};
    case Group::Bn254G2: return {128, 255};
    case Group::Bls12G1: return {96, 256};
    default: return {192, 256};
  }
}

struct BasesEntry {
  DevBuf d;
  size_t n = 0;
  Group group = Group::Bn254G1;
  bool g2_gen0 = false;  // BLS12-381 G2: point 0 is the generator (so point 1 is [tau]2 of a KZG setup)
  uint32_t table_c = 0;  // != 0: d holds W = ceil(255/c) windows of n points: 2^(c*w) * P_i at w*n + i
  // a 4096-point BLS12-381 G1 monomial setup used for EIP-7594 cell proofs (kzg_cells.cu): its FK20 table, 64 x 128 native
  // affine points, built on the handle's first such call and freed with it
  OnceTable fk20;
};

// a snarkjs Groth16 key loaded by b200zk_groth16_zkey_load (zkey.cu): its columns and key terms live in ctx->bases under
// the handles below; the A and B coefficient rows are one CSR over 2 * domainSize rows (A's rows, then B's)
struct ZkeyEntry {
  uint32_t n_vars = 0, n_public = 0, log_n = 0, nnz = 0;
  uint64_t col[5] = {0, 0, 0, 0, 0};  // A, B1, B2, C (signals n_public+1 ..), H
  uint64_t terms_g1 = 0, terms_g2 = 0;  // alpha1, beta1, delta1 | beta2, delta2
  DevBuf row_ptr, sig, val;  // CSR: 2 * domainSize + 1 offsets, nnz signal indices, nnz values (coef * R^2 mod r)
  DevBuf one;                // the canonical 1: the quotient step's zinv (no division by Z on the odd coset)
  uint8_t omega[32] = {};    // w_2n, canonical little-endian: the odd coset's generator
  std::vector<uint8_t> vk;   // alpha1 | beta2 | gamma2 | delta2 | IC, EIP-196/197 bytes
};

// a snarkjs PLONK key loaded by b200zk_plonk_zkey_load (plonk.cu): PTau lives in ctx->bases under `ptau`; the rest is
// the key's own (all Fr values Montgomery)
struct PlonkEntry {
  uint32_t n_vars = 0, n_public = 0, log_n = 0, n_additions = 0, n_constraints = 0;
  uint64_t ptau = 0;
  DevBuf coef;     // Qm Ql Qr Qo Qc S1 S2 S3: domainSize coefficients each
  DevBuf coset;    // the same 8, then L1, on the coset 5 <w_4n>: 4 domainSize values each
  DevBuf sigma_h;  // S1 S2 S3 on the domain <w_n>
  DevBuf maps;     // the A, B, C maps: nConstraints u32 each
  DevBuf adds;     // the additions in level order: uint4 (dst, s1, s2, 0) each, then f1 and f2 as two Fr arrays
  std::vector<uint32_t> level_off;  // additions of level k are [level_off[k], level_off[k + 1])
  DevBuf consts;   // the constants of plonk.cu's kC* slots, then the verifying key's 736 bytes
  std::vector<uint8_t> vk;
};

}  // namespace b200zk

struct b200zk_ctx {
  int device = 0;
  int sm_count = 132;
  cudaStream_t stream = nullptr;
  std::string last_error;
  uint64_t launches = 0;
  uint32_t msm_window = 0;
  uint32_t msm_chunks = 0;   // chunk count of the MSM schedule; 0 = automatic
  cudaStream_t stream_upload = nullptr;  // copy stream: host scalars of a chunked MSM upload on it, one chunk ahead of the kernels
  cudaEvent_t ev_in = nullptr;
  cudaEvent_t ev_up[64] = {};  // upload k of a chunked MSM has landed (recorded on stream_upload, waited on by the caller's stream)
  b200zk::SortWorkspace sort;
  b200zk::DevBuf ws_totals, ws_bitpart;
  b200zk::DevBuf ws_g16[4];   // b200zk_groth16_commit: staged A/B/C evaluations (host inputs) and the 768-byte partial block
  b200zk::DevBuf ws_zinv;     // 1/(5^n - 1) of the last quotient domain, canonical limbs (cached per log_n)
  uint32_t zinv_log_n = 0xffffffffu;
  // cudaFuncSetAttribute (opt-in to > 48 KiB dynamic shared memory) is per DEVICE: remembered per context, not per process
  bool attr_sort = false, attr_acc = false, attr_ntt512 = false, attr_ntt256 = false, attr_kzg = false, attr_kzg_cells = false;
  // tables built once per context on first use (once_table):
  //   kzg_roots (bls381.cu): the EIP-4844 blob domain's 4096 roots of unity in bit-reversed order, then 1/4096 (Fr381 Montgomery)
  //   kzg_cells_tw (kzg_cells.cu): w^i for the 8192nd root w, i < 8192, then 1/4096 (Fr381 Montgomery)
  //   secp_gtab (secp256k1.cu): d G for d = 1 .. 4095 as affine secp256k1 points (256 KB)
  //   p256_gtab (secp256r1.cu): the same table for the P-256 generator (affine, Montgomery form, 256 KB)
  b200zk::OnceTable kzg_roots, kzg_cells_tw, secp_gtab, p256_gtab;
  b200zk::DevBuf ws_kzg;      // EIP-4844 / EIP-7594 proofs and cells: blobs, z, quotients, partial sums and encoded results of one call
  b200zk::DevBuf ws_pairing;  // BLS12-381 pairing checks and KZG verification (bls_pairing.cu): inputs, points, lines, Miller values;
                              // also the inputs and outputs of the EIP-2537 (bls_ops.cu), ECRECOVER (secp256k1.cu),
                              // P256VERIFY (secp256r1.cu) and MODEXP (modexp.cu: operand bytes, item list, outputs) batches
  bool profiling = false;
  float phase_ms[6] = {0, 0, 0, 0, 0, 0};
  cudaEvent_t ev[8] = {};
  cudaEvent_t ev_plonk[6] = {};  // with profiling: the round boundaries of the last b200zk_plonk_zkey_prove
  float plonk_round_ms[5] = {0, 0, 0, 0, 0};
  // grow-only workspaces (every DevBuf, OnceTable and BasesEntry frees itself when the context is deleted)
  b200zk::DevBuf ws_buckets, ws_chunkS, ws_chunkV, ws_result, ws_points, ws_scalars, ws_ntt, ws_misc, ws_out, ws_segbucket;
  // 2^28-th primitive root of unity of Fr the NTT derives its domain generators from (canonical limbs).
  // Default = ark-poly / gnark-crypto 5^((r-1)/2^28); halo2curves uses 7^((r-1)/2^28) (b200zk_set_ntt_root).
  uint32_t ntt_root[8] = {0x725b19f0u, 0x9bd61b6eu, 0x41112ed4u, 0x402d111eu, 0x8ef62abcu, 0x00e0a7ebu, 0xa58a7e85u, 0x2a3c09f0u};
  uint64_t ntt_root_id = 0;  // 0 = default; else a hash of ntt_root (part of the twiddle cache key)
  std::map<uint64_t, b200zk::TwiddleSet> twiddles;
  std::map<uint64_t, b200zk::BasesEntry> bases;
  std::map<uint64_t, b200zk::ZkeyEntry> zkeys;  // handles share next_handle with the bases
  b200zk::DevBuf ws_zkey;     // b200zk_groth16_zkey_prove: witness, evaluations and the evaluation's carries
  std::map<uint64_t, b200zk::PlonkEntry> plonk_keys;  // b200zk_plonk_zkey_load; handles share next_handle too
  b200zk::DevBuf ws_plonk;    // b200zk_plonk_zkey_prove: witness, polynomials, coset values, scans, challenges, proof
  uint64_t next_handle = 1;
  uint8_t* h_pinned = nullptr;  // 4 KiB pinned staging for results / flags
};

namespace b200zk {

inline int fail(b200zk_ctx* ctx, int status, const char* what, cudaError_t e = cudaSuccess) {
  if (ctx) {
    ctx->last_error = what;
    if (e != cudaSuccess) { ctx->last_error += ": "; ctx->last_error += cudaGetErrorString(e); }
  }
  return status;
}

#define B2_CUDA(ctx, expr)                                                      \
  do {                                                                          \
    cudaError_t _e = (expr);                                                    \
    if (_e != cudaSuccess) return b200zk::fail(ctx, _e == cudaErrorMemoryAllocation ? B200ZK_ERR_OOM : B200ZK_ERR_CUDA, #expr, _e); \
  } while (0)

#define B2_TRY(expr)                        \
  do {                                      \
    int _s = (expr);                        \
    if (_s > B200ZK_OK_INFINITY) return _s; \
  } while (0)

inline int ensure(b200zk_ctx* ctx, DevBuf& b, size_t bytes) {
  if (bytes <= b.cap) return B200ZK_OK;
  // never free a buffer that queued kernels may still read
  B2_CUDA(ctx, cudaDeviceSynchronize());
  if (b.p) { cudaFree(b.p); b.p = nullptr; b.cap = 0; }
  size_t want = bytes + bytes / 8;
  cudaError_t e = cudaMalloc(&b.p, want);
  if (e != cudaSuccess) { cudaGetLastError(); want = bytes; e = cudaMalloc(&b.p, want); }
  if (e != cudaSuccess) { cudaGetLastError(); b.p = nullptr; return fail(ctx, B200ZK_ERR_OOM, "cudaMalloc workspace", e); }
  b.cap = want;
  return B200ZK_OK;
}

// Every extern "C" entry runs on the context's device, whatever device is current on the calling thread (two
// contexts in one process, or a torch current device that differs from the context's), and restores it on exit.
struct DeviceGuard {
  int prev = -1;
  bool switched = false;
  explicit DeviceGuard(const b200zk_ctx* ctx) {
    if (!ctx) return;
    if (cudaGetDevice(&prev) != cudaSuccess) { cudaGetLastError(); prev = -1; }
    if (prev != ctx->device) { switched = cudaSetDevice(ctx->device) == cudaSuccess; if (!switched) cudaGetLastError(); }
  }
  ~DeviceGuard() { if (switched && prev >= 0) cudaSetDevice(prev); }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;
};

// NVTX range over one library phase (SURVEY.md section 5: the reference's tracing spans around proving, e.g.
// crates/prover/src/prover.rs:106-118; here per C-ABI call and per MSM / NTT phase)
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
  NvtxRange(const NvtxRange&) = delete;
  NvtxRange& operator=(const NvtxRange&) = delete;
};

inline cudaStream_t pick_stream(b200zk_ctx* ctx, void* stream) { return stream ? (cudaStream_t)stream : ctx->stream; }

// carves one call's buffers out of a workspace: run the same sequence of take() once with base = nullptr to size it
struct Carve {
  uint8_t* base = nullptr;
  size_t off = 0;
  template <class T> T* take(size_t count) {
    off = (off + 255) & ~(size_t)255;
    T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
    off += count * sizeof(T);
    return p;
  }
};

// runs layout(Carve&) once to size the call's buffers, grows ws to fit, then runs it again over ws.p
template <class Layout> int carve(b200zk_ctx* ctx, DevBuf& ws, Layout&& layout) {
  Carve c;
  layout(c);
  B2_TRY(ensure(ctx, ws, c.off + 256));
  c = Carve{(uint8_t*)ws.p, 0};
  layout(c);
  return B200ZK_OK;
}

// The table t (bytes long) on stream st: the first call allocates it, enqueues enqueue_build(void* table) (an int status)
// and records t.ready behind it; later calls wait on t.ready.  A failed build leaves t unbuilt, so the next call builds it
// again.  Without an event the build is synchronised here instead.
template <class Build>
int once_table(b200zk_ctx* ctx, OnceTable& t, size_t bytes, cudaStream_t st, Build&& enqueue_build, const void** out) {
  if (!t.built) {
    B2_TRY(ensure(ctx, t.buf, bytes));
    B2_TRY(enqueue_build(t.buf.p));
    if (!t.ready && cudaEventCreateWithFlags(&t.ready, cudaEventDisableTiming) != cudaSuccess) { cudaGetLastError(); t.ready = nullptr; }
    if (t.ready) B2_CUDA(ctx, cudaEventRecord(t.ready, st));
    else B2_CUDA(ctx, cudaStreamSynchronize(st));
    t.built = true;
  } else if (t.ready) {
    B2_CUDA(ctx, cudaStreamWaitEvent(st, t.ready, 0));
  }
  *out = t.buf.p;
  return B200ZK_OK;
}

// the resident bases behind handle (of group g), or nullptr after failing with msg
inline BasesEntry* find_bases(b200zk_ctx* ctx, uint64_t handle, const char* msg) {
  auto it = ctx->bases.find(handle);
  if (it != ctx->bases.end()) return &it->second;
  fail(ctx, B200ZK_ERR_INVALID_ARG, msg);
  return nullptr;
}
inline BasesEntry* find_bases(b200zk_ctx* ctx, uint64_t handle, Group g, const char* msg) {
  BasesEntry* e = find_bases(ctx, handle, msg);
  if (!e || e->group == g) return e;
  fail(ctx, B200ZK_ERR_INVALID_ARG, msg);
  return nullptr;
}

// takes ownership of a filled entry under a new handle
inline int register_bases(b200zk_ctx* ctx, BasesEntry&& e, uint64_t* handle) {
  *handle = ctx->next_handle++;
  ctx->bases.emplace(*handle, std::move(e));
  return B200ZK_OK;
}

// pair_offsets of `count` >= 1 checks: first entry 0, never decreasing
inline int check_offsets(b200zk_ctx* ctx, const uint32_t* offsets, size_t count, const char* what) {
  if (offsets[0] != 0) return fail(ctx, B200ZK_ERR_INVALID_ARG, (std::string(what) + ": pair_offsets[0] must be 0").c_str());
  for (size_t i = 0; i < count; ++i)
    if (offsets[i + 1] < offsets[i]) return fail(ctx, B200ZK_ERR_INVALID_ARG, (std::string(what) + ": pair_offsets must be non-decreasing").c_str());
  return B200ZK_OK;
}

// every kernel launch in the library goes through this macro so gpu_launches is a count, not a guess
#define B2_LAUNCH(ctx, kernel, grid, block, smem, st, ...)                                   \
  do {                                                                                       \
    kernel<<<(grid), (block), (smem), (st)>>>(__VA_ARGS__);                                  \
    (ctx)->launches++;                                                                       \
    cudaError_t _e = cudaGetLastError();                                                     \
    if (_e != cudaSuccess) return b200zk::fail(ctx, B200ZK_ERR_CUDA, "launch " #kernel, _e); \
  } while (0)

// 32-byte element as two 128-bit words: every field element moves through HBM as LDG.128/STG.128 pairs
template <class F> B2_D F load_fe(const void* base, size_t index) {
  const uint4* p = reinterpret_cast<const uint4*>(base) + 2 * index;
  uint4 lo = p[0], hi = p[1];
  F r;
  r.v[0] = lo.x; r.v[1] = lo.y; r.v[2] = lo.z; r.v[3] = lo.w;
  r.v[4] = hi.x; r.v[5] = hi.y; r.v[6] = hi.z; r.v[7] = hi.w;
  return r;
}
template <class F> B2_D F load_fe_nc(const void* base, size_t index) {  // read-only path
  const uint4* p = reinterpret_cast<const uint4*>(base) + 2 * index;
  uint4 lo = __ldg(p), hi = __ldg(p + 1);
  F r;
  r.v[0] = lo.x; r.v[1] = lo.y; r.v[2] = lo.z; r.v[3] = lo.w;
  r.v[4] = hi.x; r.v[5] = hi.y; r.v[6] = hi.z; r.v[7] = hi.w;
  return r;
}
template <class F> B2_D void store_fe(void* base, size_t index, const F& a) {
  uint4* p = reinterpret_cast<uint4*>(base) + 2 * index;
  p[0] = make_uint4(a.v[0], a.v[1], a.v[2], a.v[3]);
  p[1] = make_uint4(a.v[4], a.v[5], a.v[6], a.v[7]);
}

// field-generic element I/O at "slot" granularity: slot = index of a 32-byte word
B2_D Fq load_field(const void* base, size_t slot, const Fq*) { return load_fe<Fq>(base, slot); }
B2_D Fq2 load_field(const void* base, size_t slot, const Fq2*) { return {load_fe<Fq>(base, 2 * slot), load_fe<Fq>(base, 2 * slot + 1)}; }
B2_D Fq load_field_nc(const void* base, size_t slot, const Fq*) { return load_fe_nc<Fq>(base, slot); }
B2_D Fq2 load_field_nc(const void* base, size_t slot, const Fq2*) { return {load_fe_nc<Fq>(base, 2 * slot), load_fe_nc<Fq>(base, 2 * slot + 1)}; }
B2_D void store_field(void* base, size_t slot, const Fq& a) { store_fe<Fq>(base, slot, a); }
B2_D void store_field(void* base, size_t slot, const Fq2& a) { store_fe<Fq>(base, 2 * slot, a.c0); store_fe<Fq>(base, 2 * slot + 1, a.c1); }

// 48-byte (Fp381) elements: three 128-bit words
B2_D Fp381 load_field(const void* base, size_t slot, const Fp381*) {
  const uint4* p = reinterpret_cast<const uint4*>(base) + 3 * slot;
  uint4 a = p[0], b = p[1], c = p[2];
  Fp381 r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w; r.v[8] = c.x; r.v[9] = c.y; r.v[10] = c.z; r.v[11] = c.w;
  return r;
}
B2_D Fp381 load_field_nc(const void* base, size_t slot, const Fp381*) {
  const uint4* p = reinterpret_cast<const uint4*>(base) + 3 * slot;
  uint4 a = __ldg(p), b = __ldg(p + 1), c = __ldg(p + 2);
  Fp381 r;
  r.v[0] = a.x; r.v[1] = a.y; r.v[2] = a.z; r.v[3] = a.w; r.v[4] = b.x; r.v[5] = b.y; r.v[6] = b.z; r.v[7] = b.w; r.v[8] = c.x; r.v[9] = c.y; r.v[10] = c.z; r.v[11] = c.w;
  return r;
}
B2_D void store_field(void* base, size_t slot, const Fp381& a) {
  uint4* p = reinterpret_cast<uint4*>(base) + 3 * slot;
  p[0] = make_uint4(a.v[0], a.v[1], a.v[2], a.v[3]); p[1] = make_uint4(a.v[4], a.v[5], a.v[6], a.v[7]); p[2] = make_uint4(a.v[8], a.v[9], a.v[10], a.v[11]);
}

template <class F> B2_D Affine<F> load_affine_nc(const void* base, size_t i) {
  return {load_field_nc(base, 2 * i, (const F*)nullptr), load_field_nc(base, 2 * i + 1, (const F*)nullptr)};
}
template <class F> B2_D void store_affine(void* base, size_t i, const Affine<F>& p) {
  store_field(base, 2 * i, p.x); store_field(base, 2 * i + 1, p.y);
}
template <class F> B2_D XYZZ<F> load_xyzz(const void* base, size_t i) {
  const F* t = nullptr;
  return {load_field(base, 4 * i, t), load_field(base, 4 * i + 1, t), load_field(base, 4 * i + 2, t), load_field(base, 4 * i + 3, t)};
}
template <class F> B2_D void store_xyzz(void* base, size_t i, const XYZZ<F>& p) {
  store_field(base, 4 * i, p.x); store_field(base, 4 * i + 1, p.y); store_field(base, 4 * i + 2, p.zz); store_field(base, 4 * i + 3, p.zzz);
}
template <class F> struct FieldBytes;
template <> struct FieldBytes<Fq> { static constexpr size_t value = 32; };
template <> struct FieldBytes<Fq2> { static constexpr size_t value = 64; };
template <> struct FieldBytes<Fp381> { static constexpr size_t value = 48; };
template <class F> struct ScalarBits { static constexpr uint32_t value = 255; };  // BN254: r < 2^254, + 1 for the recoding's carry
template <> struct ScalarBits<Fp381> { static constexpr uint32_t value = 256; };     // BLS12-381: r < 2^255
template <class F> struct IsFq2 { static constexpr bool value = false; };
template <> struct IsFq2<Fq2> { static constexpr bool value = true; };

// internal cross-TU entry points
// table_c != 0: d_points is a precomputed window table with `table_stride` points per window
// h_scalars != nullptr: the scalars are in (pinned) host memory and are uploaded chunk by chunk inside the pipeline
int msm_run_g1(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n, uint32_t flags, cudaStream_t st, void* d_partial, uint32_t table_c = 0, size_t table_stride = 0, const void* h_scalars = nullptr, int sort_mode = 0);
int msm_run_g2(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n, uint32_t flags, cudaStream_t st, void* d_partial, uint32_t table_c = 0, size_t table_stride = 0, const void* h_scalars = nullptr, int sort_mode = 0);
int msm_run_bls(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n, uint32_t flags, cudaStream_t st, void* d_partial, uint32_t table_c = 0, size_t table_stride = 0, const void* h_scalars = nullptr, int sort_mode = 0);
int msm_precompute_bls(b200zk_ctx* ctx, const void* d_bases, size_t n, uint32_t c, void* d_table, cudaStream_t st);
int msm_encode_bls(b200zk_ctx* ctx, const void* d_partials, size_t count, uint32_t flags, cudaStream_t st, void* d_out);
// compressed (48 B, ZCash format) or uncompressed (96 B big-endian x | y) G1 points -> native affine; status[0] = first index with a coordinate >= p,
// status[1] = first index not on the curve / with malformed flag bits (each n when none)
int bls_points_to_native(b200zk_ctx* ctx, const void* d_in, void* d_native, size_t n, bool compressed, cudaStream_t st);
// first index of a 32-byte scalar (big-endian, or little-endian limbs) >= the BLS12-381 group order among n, or n
int bls_scalars_check(b200zk_ctx* ctx, const void* d_scalars, size_t n, bool big_endian, cudaStream_t st, size_t* bad_index);
// the same check enqueued on st without a synchronisation: *d_bad, set to n by the caller, ends as the first such index
int bls_scalars_check_enqueue(b200zk_ctx* ctx, const void* d_scalars, size_t n, bool big_endian, cudaStream_t st, unsigned long long* d_bad);
int msm_precompute_g1(b200zk_ctx* ctx, const void* d_bases, size_t n, uint32_t c, void* d_table, cudaStream_t st);
int msm_precompute_g2(b200zk_ctx* ctx, const void* d_bases, size_t n, uint32_t c, void* d_table, cudaStream_t st);
uint32_t precompute_window(size_t n);
int msm_encode_g1(b200zk_ctx* ctx, const void* d_partials, size_t count, uint32_t flags, cudaStream_t st, void* d_out);
int msm_encode_g2(b200zk_ctx* ctx, const void* d_partials, size_t count, uint32_t flags, cudaStream_t st, void* d_out);
int points_be_to_native(b200zk_ctx* ctx, const void* d_be, void* d_native, size_t n, bool g2, cudaStream_t st);
int ntt_run(b200zk_ctx* ctx, void* d_data, uint32_t log_n, uint32_t flags, const uint8_t* coset_gen, cudaStream_t st);
int ntt_set_root(b200zk_ctx* ctx, const uint8_t* root_le);
// out[i] = (a[i]*b[i] - c[i]) * zinv, zinv read from device memory (canonical limbs)
int fr_quotient_dev(b200zk_ctx* ctx, const void* d_a, const void* d_b, const void* d_c, void* d_out, size_t n, const uint32_t* d_zinv_canonical, cudaStream_t st);
// *d_zinv = device pointer to 1/(5^(2^log_n) - 1) (canonical limbs), computed once per log_n on `st`
int fr_coset_zinv_dev(b200zk_ctx* ctx, uint32_t log_n, cudaStream_t st, const uint32_t** d_zinv);
// the key-term pointers of a b200zk_groth16_zk after checking its handles and r, s (groth16.cu)
int groth16_zk_terms(b200zk_ctx* ctx, const b200zk_groth16_zk* zk, const void** g1, const void** g2);
// exclusive scan of G counts (seg = 0) into out[0..G], out[G] = the total; cursor, if given, receives out[0..G) too;
// tsum: one word per 2048 values (msm.cu)
int exclusive_scan(b200zk_ctx* ctx, cudaStream_t st, const uint32_t* in, const uint32_t* aux, size_t G, uint32_t seg, uint32_t* tsum,
                   uint32_t* out, uint32_t* cursor = nullptr);
int groth16_commit_partials(b200zk_ctx* ctx, const b200zk_groth16_pk* pk, const void* witness, void* a_evals, void* b_evals, void* c_evals,
                            uint32_t flags, cudaStream_t st, void* d_partials);
// d_partials: count blocks of 768 B (A | B1 | B2 | L | H as XYZZ); d_out: proof A|B2|C (256 B) | B1 (64 B) | 4 x u32 is_infinity (A, B2, C, B1)
int groth16_assemble_dev(b200zk_ctx* ctx, const void* d_partials, size_t count, cudaStream_t st, void* d_out);
// same blocks with the key terms (g1: alpha, beta, delta; g2: beta, delta; native affine) and the blinding scalars r, s
// (canonical LE, < the group order); d_out: proof A|B2|C (256 B) | 3 x u32 is_infinity (A, B2, C)
int groth16_assemble_zk_dev(b200zk_ctx* ctx, const void* d_partials, size_t count, const void* d_g1_terms, const void* d_g2_terms,
                            const uint8_t r_le[32], const uint8_t s_le[32], cudaStream_t st, void* d_out);
int bn254_g1_add_batch(b200zk_ctx* ctx, const uint8_t* a, const uint8_t* b, size_t count, uint8_t* out, uint8_t* status);
int bn254_g1_mul_batch(b200zk_ctx* ctx, const uint8_t* points, const uint8_t* scalars, size_t count, uint8_t* out, uint8_t* status);
int bn254_pairing_check_batch(b200zk_ctx* ctx, const uint8_t* pairs, const uint32_t* pair_offsets, size_t count, uint8_t* result, uint8_t* status);
// EIP-4844 (bls381.cu): the Fiat-Shamir challenge of one blob, and y = p(z) of n blobs on the device (the quotient goes to
// d_q, n x 4096 x 32 bytes of scratch).  The digest-to-field reduction, hash_to_bls_field, is in cell_batch.h.
void kzg_challenge(const uint8_t* blob, const uint8_t commitment[48], uint8_t z_be[32]);
int kzg_eval_run(b200zk_ctx* ctx, const uint8_t* d_blobs, const uint8_t* d_z, size_t n, void* d_q, uint8_t* d_y, cudaStream_t st);
// the setup handle of a KZG call: a BLS12-381 G1 handle of exactly 4096 points, else status 4 naming `what`
int kzg_setup(b200zk_ctx* ctx, uint64_t handle, const char* what, BasesEntry** e);
// one 4096-point MSM per blob over the setup (scalars n x 4096 x 32 bytes): XYZZ partial sums 192 B apart, each encoded into
// its own 128-byte slot of enc (the 48-byte compressed point first)
int kzg_msms(b200zk_ctx* ctx, const BasesEntry& e, const uint8_t* scalars, size_t n, uint32_t flags, uint8_t* partials, uint8_t* enc, cudaStream_t st);
// EIP-7594 (kzg_cells.cu): the 128 cells of n blobs (checked < r), n x 8192 x 32 bytes big-endian; and from the challenge
// r (32-byte big-endian, < r) the scalars of the batched cell-proof check, canonical little-endian limbs: s_proof (128 n)
// = r^k, s_lin (129 n) = the n commitments' sum_c r^(128 b + c), then r^k h_k^64; s_setup (4096) = sum_k r^k I_k on the
// bit-reversed roots.  Scratch: weights 65 x 32 bytes, partial n x 64 x 32 bytes
int kzg_cells_run(b200zk_ctx* ctx, const uint8_t* d_blobs, size_t n, uint8_t* d_cells, cudaStream_t st);
int kzg_cell_scalars_run(b200zk_ctx* ctx, const uint8_t* d_blobs, size_t n, const uint8_t* d_r_be, void* d_weights, void* d_partial,
                         void* d_s_proof, void* d_s_lin, void* d_s_setup, cudaStream_t st);
// The same scalars for n arbitrary cells (b200zk_kzg_verify_cells, cells n x 2048 bytes big-endian, checked < r), from the
// host's groupings (cell_batch.h) on the device: s_proof (n) = r^k; s_lin (n_commit + n) = each deduplicated commitment's
// sum of r^k over its cells, then r^k h_k^64; s_setup (4096) as above.  Scratch: rpow n x 32 bytes, partial n_cols x 64
// x 32 bytes
struct VCellsMeta {
  size_t n = 0, n_commit = 0, n_cols = 0;
  const uint32_t* idx = nullptr;         // n: the cell index of each cell
  const uint32_t* commit_off = nullptr;  // n_commit + 1, into by_commit (n)
  const uint32_t* by_commit = nullptr;
  const uint32_t* column_off = nullptr;  // n_cols + 1, into by_column (n); columns (n_cols): the cell indices that occur
  const uint32_t* by_column = nullptr;
  const uint32_t* columns = nullptr;
};
int kzg_vcells_scalars_run(b200zk_ctx* ctx, const uint8_t* d_cells, const VCellsMeta& m, const uint8_t* d_r_be, void* d_rpow, void* d_partial,
                           void* d_s_proof, void* d_s_lin, void* d_s_setup, cudaStream_t st);

// every element of n_blobs big-endian blobs, and of the n_extra z values right behind them, < r; else status 2 naming
// `what` and the first offending blob and element (or z)
inline int check_blobs(b200zk_ctx* ctx, const uint8_t* d_blobs, size_t n_blobs, size_t n_extra, cudaStream_t st, const char* what) {
  constexpr size_t kElems = 4096;  // FIELD_ELEMENTS_PER_BLOB
  const size_t elems = n_blobs * kElems;
  size_t bad = elems + n_extra;
  B2_TRY(bls_scalars_check(ctx, d_blobs, elems + n_extra, true, st, &bad));
  if (bad >= elems + n_extra) return B200ZK_OK;
  char msg[160];
  if (bad < elems) snprintf(msg, sizeof msg, "%s: blob %zu, element %zu is >= the BLS12-381 group order", what, bad / kElems, bad % kElems);
  else snprintf(msg, sizeof msg, "%s: z of blob %zu is >= the BLS12-381 group order", what, bad - elems);
  return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, msg);
}

}  // namespace b200zk
