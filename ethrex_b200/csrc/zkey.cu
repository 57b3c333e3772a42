// zkey.cu -- Groth16 from circom artifacts: a snarkjs .zkey loaded once into HBM, each .wtns witness proved in one call
// (b200zk_groth16_zkey_*; formats in include/b200zk.h, parser in zkey_parse.cpp).
//
//   load    parse (host) -> columns A, B1, B2, C, H and the key terms uploaded as resident bases, every coordinate checked
//           < q and every point on its curve -> the section-4 records checked and sorted into one CSR by row
//           (histogram zkey_coef_count, exclusive_scan of msm.cu, scatter zkey_coef_scatter) -> optional window tables
//   prove   witness range check (zkey_wtns_check) -> a = A w, b = B w (zkey_eval + zkey_eval_fixup) -> c = a o b ->
//           per column iNTT and NTT on the odd coset w_2n <w_n> -> P = a b - c (fr_quotient with zinv = 1) ->
//           the MSMs of groth16_commit_partials with H over P -> the key terms and r, s blinding (groth16_assemble_zk_dev)
//
// The sparse evaluation balances work over nonzeros, not rows: circom rows are skewed (most hold a few terms, a few hold
// thousands).  Thread t sums the fixed slice [16 t, 16 t + 16) of the CSR's values.  A row that starts and ends inside
// the slice is stored directly; the first row of a slice that began in an earlier slice leaves its partial sum in
// carry_first[t]; the last row, when it continues past the slice, leaves carry_last[t] and lists t as the row's owner.
// One warp per owner then adds the owner's carry_last to the carry_first of every slice the row covers.
#include "common.cuh"
#include "zkey_parse.h"

#include <cstring>
#include <vector>

namespace b200zk {

static constexpr uint32_t kSlice = 16;  // nonzeros per thread of zkey_eval

struct Limbs8 { uint32_t v[8]; };

// ---- load ------------------------------------------------------------------------------------------------------------
// min index of a 32-byte Montgomery word >= q among n (a coordinate out of range)
__global__ void __launch_bounds__(256) zkey_words_check(const void* words, size_t n, unsigned long long* bad) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    Fq v = load_fe_nc<Fq>(words, i), m = Fq::modulus(), t;
    if (!detail::sub8(t.v, v.v, m.v)) atomicMin(bad, (unsigned long long)i);
  }
}

// the records' check (zkey_coef_check, shared with the host parser) and the histogram of their rows
// (matrix * domain + constraint); bad = min index of a failing record
__global__ void __launch_bounds__(256) zkey_coef_count(const uint32_t* rec, size_t n, uint32_t domain, uint32_t n_vars, uint32_t* count,
                                                       unsigned long long* bad) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t w[11];
#pragma unroll
    for (int k = 0; k < 11; ++k) w[k] = __ldg(rec + 11 * i + k);
    if (zkey_coef_check(w, domain, n_vars) != ZKEY_COEF_OK) { atomicMin(bad, (unsigned long long)i); continue; }
    atomicAdd(count + (size_t)w[0] * domain + w[1], 1u);
  }
}

// every record into its row's next free place; the order inside a row does not matter (the row is a sum)
__global__ void __launch_bounds__(256) zkey_coef_scatter(const uint32_t* rec, size_t n, uint32_t domain, uint32_t* cursor, uint32_t* sig, void* val) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const uint32_t* w = rec + 11 * i;
    const uint32_t pos = atomicAdd(cursor + (size_t)__ldg(w) * domain + __ldg(w + 1), 1u);
    sig[pos] = __ldg(w + 2);
    Fr v;
#pragma unroll
    for (int k = 0; k < 8; ++k) v.v[k] = __ldg(w + 3 + k);
    store_fe<Fr>(val, pos, v);
  }
}

// out = w_(2^log_2n) = root^(2^(28 - log_2n)), canonical limbs, from a 2^28-th root of unity (canonical)
__global__ void zkey_omega(Limbs8 root, uint32_t log_2n, uint32_t* out) {
  if (blockIdx.x || threadIdx.x) return;
  Fr g;
#pragma unroll
  for (int k = 0; k < 8; ++k) g.v[k] = root.v[k];
  g = Fr::to_mont(g);
  for (uint32_t i = log_2n; i < 28; ++i) g = Fr::sqr(g);
  g = Fr::from_mont(g);
#pragma unroll
  for (int k = 0; k < 8; ++k) out[k] = g.v[k];
}

// n Montgomery Fq words -> 32-byte big-endian canonical values (the verifying key's EIP-196/197 bytes)
__global__ void __launch_bounds__(128) zkey_words_to_be(const void* words, size_t n, uint8_t* be) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    Fq v = Fq::from_mont(load_fe_nc<Fq>(words, i));
    for (int k = 0; k < 8; ++k) {
      const uint32_t limb = v.v[7 - k];
      be[32 * i + 4 * k] = (uint8_t)(limb >> 24); be[32 * i + 4 * k + 1] = (uint8_t)(limb >> 16);
      be[32 * i + 4 * k + 2] = (uint8_t)(limb >> 8); be[32 * i + 4 * k + 3] = (uint8_t)limb;
    }
  }
}

// ---- prove -----------------------------------------------------------------------------------------------------------
// min index of a witness value >= r among n (canonical little-endian)
__global__ void __launch_bounds__(256) zkey_wtns_check(const void* wit, size_t n, unsigned long long* bad) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    Fr v = load_fe_nc<Fr>(wit, i), m = Fr::modulus(), t;
    if (!detail::sub8(t.v, v.v, m.v)) atomicMin(bad, (unsigned long long)i);
  }
}

// the row holding nonzero e: the last r with row_ptr[r] <= e (rows below it may be empty)
B2_D uint32_t zkey_row_of(const uint32_t* row_ptr, uint32_t rows, uint32_t e) {
  uint32_t lo = 0, hi = rows;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(row_ptr + mid) <= e) lo = mid; else hi = mid;
  }
  return lo;
}

// out[row] = sum_e val[e] * wit[sig[e]] (Montgomery products of coef * R^2 and a canonical value: the Montgomery form of
// coef * w) for the rows that start and end inside a slice; carries for the others (see the file comment)
__global__ void __launch_bounds__(256) zkey_eval(const uint32_t* row_ptr, uint32_t rows, const uint32_t* sig, const void* val, const void* wit,
                                                 uint32_t nnz, void* out, void* carry_first, void* carry_last, uint32_t* owners, uint32_t* n_owners) {
  const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (t * kSlice >= nnz) return;
  const uint32_t e0 = (uint32_t)(t * kSlice), e1 = nnz - e0 < kSlice ? nnz : e0 + kSlice;
  uint32_t r = zkey_row_of(row_ptr, rows, e0), rs = __ldg(row_ptr + r), re = __ldg(row_ptr + r + 1);
  Fr acc = Fr::zero();
  for (uint32_t e = e0; e < e1; ++e) {
    while (e == re) {  // row r ends inside the slice (empty rows in between are stored as zero)
      if (rs < e0) store_fe<Fr>(carry_first, t, acc); else store_fe<Fr>(out, r, acc);
      acc = Fr::zero();
      ++r; rs = re; re = __ldg(row_ptr + r + 1);
    }
    acc = Fr::add(acc, Fr::mul(load_fe_nc<Fr>(val, e), load_fe_nc<Fr>(wit, __ldg(sig + e))));
  }
  if (rs < e0) store_fe<Fr>(carry_first, t, acc);  // began in an earlier slice (and may run on past this one)
  else if (re <= e1) store_fe<Fr>(out, r, acc);
  else { store_fe<Fr>(carry_last, t, acc); owners[atomicAdd(n_owners, 1u)] = (uint32_t)t; }
}

// one warp per owner slice t: out[row] = carry_last[t] + sum of carry_first over the later slices the row covers
__global__ void __launch_bounds__(256) zkey_eval_fixup(const uint32_t* row_ptr, uint32_t rows, const void* carry_first, const void* carry_last,
                                                       const uint32_t* owners, const uint32_t* n_owners, void* out) {
  const uint32_t lane = threadIdx.x & 31;
  const size_t warps = ((size_t)gridDim.x * blockDim.x) >> 5;
  const uint32_t count = *n_owners;
  for (size_t k = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5; k < count; k += warps) {
    const uint32_t t = owners[k];
    const uint32_t r = zkey_row_of(row_ptr, rows, t * kSlice + kSlice - 1);
    const uint32_t t_end = (__ldg(row_ptr + r + 1) - 1) / kSlice;  // the slice holding the row's last nonzero
    Fr acc = lane == 0 ? load_fe<Fr>(carry_last, t) : Fr::zero();
    for (uint32_t u = t + 1 + lane; u <= t_end; u += 32) acc = Fr::add(acc, load_fe<Fr>(carry_first, u));
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      Fr other;
#pragma unroll
      for (int w = 0; w < 8; ++w) other.v[w] = __shfl_down_sync(0xffffffffu, acc.v[w], o);
      acc = Fr::add(acc, other);
    }
    if (lane == 0) store_fe<Fr>(out, r, acc);
  }
}

static unsigned zgrid(b200zk_ctx* ctx, size_t n, unsigned block) {
  size_t g = (n + block - 1) / block, cap = (size_t)ctx->sm_count * 32;
  return (unsigned)(g < cap ? (g ? g : 1) : cap);
}

// ---- host side -------------------------------------------------------------------------------------------------------
namespace {

// the handles a load registers, erased again unless the load succeeds (a refused key leaves nothing allocated)
struct Registered {
  b200zk_ctx* ctx;
  std::vector<uint64_t> handles;
  bool keep = false;
  ~Registered() { if (!keep) for (uint64_t h : handles) ctx->bases.erase(h); }
  int add(BasesEntry&& e, uint64_t* h) { register_bases(ctx, std::move(e), h); handles.push_back(*h); return B200ZK_OK; }
};

int alloc_bases(b200zk_ctx* ctx, BasesEntry* e, size_t n, Group g) {
  e->n = n;
  e->group = g;
  B2_CUDA(ctx, cudaMalloc(&e->d.p, n * group_sizes(g).point + 32));
  return B200ZK_OK;
}

// A checked point buffer of the key: where it came from, for the refusal's message
struct PointBuf { const char* name; int section; bool g2; const void* d; size_t n; };

int load(b200zk_ctx* ctx, const uint8_t* file, size_t len, int precompute, uint64_t* key) {
  NvtxRange nvtx("b200zk:groth16_zkey_load");
  ZkeyLayout L;
  std::string err;
  int rc = zkey_parse(file, len, &L, &err);
  if (rc) return fail(ctx, rc, err.c_str());
  cudaStream_t st = ctx->stream;
  const size_t nv = L.n_vars, np = L.n_public, n = L.domain_size, nc = nv - np - 1;
  ZkeyEntry z;
  z.n_vars = L.n_vars; z.n_public = L.n_public; z.log_n = L.log_n; z.nnz = L.n_coefs;

  // ---- points: the columns, and the header's points in one small buffer (G1: alpha1 beta1 delta1 IC..; G2: beta2
  // delta2 gamma2), so that the key terms are its first 3 G1 and 2 G2 points
  BasesEntry col[5];
  static const Group kColGroup[5] = {Group::Bn254G1, Group::Bn254G1, Group::Bn254G2, Group::Bn254G1, Group::Bn254G1};
  const size_t col_n[5] = {nv, nv, nv, nc, n};
  const uint8_t* col_src[5] = {L.a, L.b1, L.b2, L.c, L.h};
  for (int k = 0; k < 5; ++k) {
    B2_TRY(alloc_bases(ctx, &col[k], col_n[k], kColGroup[k]));
    if (col_n[k]) B2_CUDA(ctx, cudaMemcpyAsync(col[k].d.p, col_src[k], col_n[k] * group_sizes(kColGroup[k]).point, cudaMemcpyHostToDevice, st));
  }
  const size_t n_g1 = 3 + np + 1;
  std::vector<uint8_t> small(n_g1 * 64 + 3 * 128);
  memcpy(&small[0], L.alpha1, 64); memcpy(&small[64], L.beta1, 64); memcpy(&small[128], L.delta1, 64);
  memcpy(&small[192], L.ic, 64 * (np + 1));
  uint8_t* g2s = &small[n_g1 * 64];
  memcpy(g2s, L.beta2, 128); memcpy(g2s + 128, L.delta2, 128); memcpy(g2s + 256, L.gamma2, 128);
  DevBuf d_small, d_flags;
  B2_CUDA(ctx, cudaMalloc(&d_small.p, small.size() + 32 * (n_g1 * 2 + 12)));  // the points, then their BE encoding
  B2_CUDA(ctx, cudaMemcpyAsync(d_small.p, small.data(), small.size(), cudaMemcpyHostToDevice, st));
  const uint8_t* ds = (const uint8_t*)d_small.p;
  const PointBuf bufs[7] = {{"header / IC", 2, false, ds, n_g1}, {"header", 2, true, ds + n_g1 * 64, 3}, {"A", 5, false, col[0].d.p, nv},
                            {"B1", 6, false, col[1].d.p, nv}, {"B2", 7, true, col[2].d.p, nv}, {"C", 8, false, col[3].d.p, nc}, {"H", 9, false, col[4].d.p, n}};
  // every coordinate < q (one flag per buffer, read back once), then every point on its curve
  B2_CUDA(ctx, cudaMalloc(&d_flags.p, 8 * 8));
  B2_CUDA(ctx, cudaMemsetAsync(d_flags.p, 0xff, 8 * 8, st));
  unsigned long long* flags = (unsigned long long*)d_flags.p;
  for (int k = 0; k < 7; ++k) {
    const size_t words = bufs[k].n * (bufs[k].g2 ? 4 : 2);
    if (words) B2_LAUNCH(ctx, zkey_words_check, zgrid(ctx, words, 256), 256, 0, st, bufs[k].d, words, flags + k);
  }
  unsigned long long* hf = (unsigned long long*)(ctx->h_pinned + 1536);
  B2_CUDA(ctx, cudaMemcpyAsync(hf, flags, 8 * 7, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  auto point_name = [&](int k, size_t i, char* msg, size_t cap, const char* what) {
    if (k == 0 && i >= 3) snprintf(msg, cap, "zkey: section 3 (IC): point %zu %s", i - 3, what);
    else if (k <= 1) snprintf(msg, cap, "zkey: section 2 (header): %s %s", k == 0 ? (i == 0 ? "alpha1" : i == 1 ? "beta1" : "delta1")
                                                                               : (i == 0 ? "beta2" : i == 1 ? "delta2" : "gamma2"), what);
    else snprintf(msg, cap, "zkey: section %d (%s): point %zu %s", bufs[k].section, bufs[k].name, i, what);
  };
  char msg[192];
  for (int k = 0; k < 7; ++k)
    if (hf[k] != ~0ull) {
      point_name(k, (size_t)(hf[k] / (bufs[k].g2 ? 4 : 2)), msg, sizeof msg, "has a coordinate >= q");
      return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, msg);
    }
  for (int k = 0; k < 7; ++k) {
    size_t bad = bufs[k].n;
    rc = bufs[k].g2 ? b200zk_g2_check_device(ctx, bufs[k].d, bufs[k].n, st, &bad) : b200zk_g1_check_device(ctx, bufs[k].d, bufs[k].n, st, &bad);
    if (rc == B200ZK_ERR_NOT_ON_CURVE) { point_name(k, bad, msg, sizeof msg, "is not on the curve"); return fail(ctx, rc, msg); }
    B2_TRY(rc);
  }

  // ---- coefficient rows: check every record, histogram, scan, scatter
  const uint32_t rows = 2 * L.domain_size;
  DevBuf d_rec, d_count, d_tsum;
  B2_CUDA(ctx, cudaMalloc(&z.row_ptr.p, 4 * ((size_t)rows + 1)));
  B2_CUDA(ctx, cudaMalloc(&z.sig.p, 4 * (size_t)L.n_coefs + 32));
  B2_CUDA(ctx, cudaMalloc(&z.val.p, 32 * (size_t)L.n_coefs + 32));
  B2_CUDA(ctx, cudaMalloc(&d_count.p, 4 * (size_t)rows * 2));  // counts, then the scatter's cursors
  B2_CUDA(ctx, cudaMalloc(&d_tsum.p, 4 * ((size_t)rows / 2048 + 2)));
  B2_CUDA(ctx, cudaMemsetAsync(d_count.p, 0, 4 * (size_t)rows, st));
  B2_CUDA(ctx, cudaMemsetAsync(flags + 7, 0xff, 8, st));
  uint32_t* count = (uint32_t*)d_count.p;
  if (L.n_coefs) {
    B2_CUDA(ctx, cudaMalloc(&d_rec.p, kZkeyCoefBytes * (size_t)L.n_coefs));
    B2_CUDA(ctx, cudaMemcpyAsync(d_rec.p, L.coefs, kZkeyCoefBytes * (size_t)L.n_coefs, cudaMemcpyHostToDevice, st));
    B2_LAUNCH(ctx, zkey_coef_count, zgrid(ctx, L.n_coefs, 256), 256, 0, st, (const uint32_t*)d_rec.p, (size_t)L.n_coefs, L.domain_size, L.n_vars, count, flags + 7);
  }
  B2_CUDA(ctx, cudaMemcpyAsync(hf + 7, flags + 7, 8, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (hf[7] != ~0ull) {  // name the first failing record from the caller's copy
    uint32_t w[11];
    memcpy(w, L.coefs + kZkeyCoefBytes * hf[7], sizeof w);
    rc = zkey_coef_error(zkey_coef_check(w, L.domain_size, L.n_vars), (size_t)hf[7], &err);
    return fail(ctx, rc, err.c_str());
  }
  B2_TRY(exclusive_scan(ctx, st, count, nullptr, rows, 0, (uint32_t*)d_tsum.p, (uint32_t*)z.row_ptr.p, count + rows));
  if (L.n_coefs)
    B2_LAUNCH(ctx, zkey_coef_scatter, zgrid(ctx, L.n_coefs, 256), 256, 0, st, (const uint32_t*)d_rec.p, (size_t)L.n_coefs, L.domain_size, count + rows,
              (uint32_t*)z.sig.p, z.val.p);

  // ---- w_2n, the constant 1 and the verifying key's bytes
  // w_2n of the preset-0 root (snarkjs / ffjavascript / ark), whatever root the context holds now: the H column is
  // defined over that doubled domain, and prove refuses any other root for its NTTs
  Limbs8 root;
  B2_TRY(b200zk_ntt_root_preset(0, (uint8_t*)root.v));
  uint8_t* d_be = (uint8_t*)d_small.p + small.size();
  B2_CUDA(ctx, cudaMalloc(&z.one.p, 64));
  B2_CUDA(ctx, cudaMemsetAsync(z.one.p, 0, 32, st));
  B2_CUDA(ctx, cudaMemsetAsync(z.one.p, 1, 1, st));
  B2_LAUNCH(ctx, zkey_omega, 1, 32, 0, st, root, L.log_n + 1, (uint32_t*)((uint8_t*)z.one.p + 32));
  B2_LAUNCH(ctx, zkey_words_to_be, zgrid(ctx, n_g1 * 2 + 12, 128), 128, 0, st, d_small.p, n_g1 * 2 + 12, d_be);
  std::vector<uint8_t> be(32 * (n_g1 * 2 + 12));
  B2_CUDA(ctx, cudaMemcpyAsync(z.omega, (uint8_t*)z.one.p + 32, 32, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(be.data(), d_be, be.size(), cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  // G2 in EIP-197 order: x_im | x_re | y_im | y_re from the native x.c0 | x.c1 | y.c0 | y.c1
  auto g2_be = [&](size_t i) {  // point i of the G2 part (0 beta2, 1 delta2, 2 gamma2)
    const uint8_t* p = &be[32 * (n_g1 * 2 + 4 * i)];
    std::vector<uint8_t> o(128);
    memcpy(&o[0], p + 32, 32); memcpy(&o[32], p, 32); memcpy(&o[64], p + 96, 32); memcpy(&o[96], p + 64, 32);
    return o;
  };
  z.vk.assign(be.begin(), be.begin() + 64);  // alpha1
  for (size_t i : {0, 2, 1}) { auto o = g2_be(i); z.vk.insert(z.vk.end(), o.begin(), o.end()); }  // beta2, gamma2, delta2
  z.vk.insert(z.vk.end(), be.begin() + 64 * 3, be.begin() + 64 * n_g1);  // IC

  // ---- register: the columns (window tables on request) and the key terms
  Registered reg{ctx, {}};
  for (int k = 0; k < 5; ++k) B2_TRY(reg.add(std::move(col[k]), &z.col[k]));
  BasesEntry t1, t2;
  B2_TRY(alloc_bases(ctx, &t1, 3, Group::Bn254G1));
  B2_TRY(alloc_bases(ctx, &t2, 2, Group::Bn254G2));
  B2_CUDA(ctx, cudaMemcpyAsync(t1.d.p, ds, 3 * 64, cudaMemcpyDeviceToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(t2.d.p, ds + n_g1 * 64, 2 * 128, cudaMemcpyDeviceToDevice, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  B2_TRY(reg.add(std::move(t1), &z.terms_g1));
  B2_TRY(reg.add(std::move(t2), &z.terms_g2));
  if (precompute)
    for (int k = 0; k < 5; ++k)
      if (col_n[k]) B2_TRY(b200zk_bases_precompute(ctx, z.col[k], 0));
  reg.keep = true;
  *key = ctx->next_handle++;
  ctx->zkeys.emplace(*key, std::move(z));
  return B200ZK_OK;
}

ZkeyEntry* find_zkey(b200zk_ctx* ctx, uint64_t key, const char* what) {
  auto it = ctx->zkeys.find(key);
  if (it != ctx->zkeys.end()) return &it->second;
  fail(ctx, B200ZK_ERR_INVALID_ARG, what);
  return nullptr;
}

int prove(b200zk_ctx* ctx, const ZkeyEntry& z, const uint8_t* wtns, size_t len, const uint8_t r[32], const uint8_t s[32], cudaStream_t st,
          uint8_t proof[256]) {
  NvtxRange nvtx("b200zk:groth16_zkey_prove");
  if (ctx->ntt_root_id != 0)
    return fail(ctx, B200ZK_ERR_INVALID_ARG, "zkey_prove: the context's NTT root is not preset 0 (the snarkjs / ark / gnark root)");
  const uint8_t* values = nullptr;
  std::string err;
  int rc = wtns_parse(wtns, len, z.n_vars, &values, &err);
  if (rc) return fail(ctx, rc, err.c_str());
  b200zk_groth16_zk zk;
  zk.g1_terms = z.terms_g1;
  zk.g2_terms = z.terms_g2;
  memcpy(zk.r, r, 32);
  memcpy(zk.s, s, 32);
  const void *g1 = nullptr, *g2 = nullptr;
  B2_TRY(groth16_zk_terms(ctx, &zk, &g1, &g2));

  const size_t n = (size_t)1 << z.log_n, nv = z.n_vars;
  const uint32_t rows = 2 * (uint32_t)n;
  const size_t slices = ((size_t)z.nnz + kSlice - 1) / kSlice;
  uint8_t *wit = nullptr, *abc = nullptr, *cf = nullptr, *cl = nullptr;
  uint32_t *owners = nullptr, *n_owners = nullptr;
  unsigned long long* bad = nullptr;
  B2_TRY(carve(ctx, ctx->ws_zkey, [&](Carve& c) {
    wit = c.take<uint8_t>(32 * nv); abc = c.take<uint8_t>(3 * 32 * n);
    cf = c.take<uint8_t>(32 * slices); cl = c.take<uint8_t>(32 * slices); owners = c.take<uint32_t>(slices);
    n_owners = c.take<uint32_t>(1); bad = c.take<unsigned long long>(1);
  }));
  B2_TRY(ensure(ctx, ctx->ws_g16[3], 1024));
  B2_TRY(ensure(ctx, ctx->ws_out, 512));
  uint8_t *a = abc, *b = abc + 32 * n, *c = abc + 64 * n;

  // ---- witness in, range-checked (the flag is read back with the proof)
  B2_CUDA(ctx, cudaMemcpyAsync(wit, values, 32 * nv, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemsetAsync(bad, 0xff, 8, st));
  B2_CUDA(ctx, cudaMemsetAsync(n_owners, 0, 4, st));
  B2_LAUNCH(ctx, zkey_wtns_check, zgrid(ctx, nv, 256), 256, 0, st, wit, nv, bad);
  // ---- a = A w, b = B w (rows past the last coefficient stay zero), c = a o b
  {
    NvtxRange nvtx_e("b200zk:zkey_eval");
    B2_CUDA(ctx, cudaMemsetAsync(a, 0, 64 * n, st));
    if (z.nnz) {
      B2_LAUNCH(ctx, zkey_eval, (unsigned)((slices + 255) / 256), 256, 0, st, (const uint32_t*)z.row_ptr.p, rows, (const uint32_t*)z.sig.p, z.val.p,
                wit, z.nnz, a, cf, cl, owners, n_owners);
      B2_LAUNCH(ctx, zkey_eval_fixup, (unsigned)ctx->sm_count * 8, 256, 0, st, (const uint32_t*)z.row_ptr.p, rows, cf, cl, owners, n_owners, a);
    }
    B2_TRY(b200zk_field_mul_device(ctx, a, b, c, n, 1, 1, st));
  }
  // ---- P = a b - c on the odd coset w_2n <w_n>: each column to coefficients and back onto the coset
  {
    NvtxRange nvtx_q("b200zk:zkey_quotient");
    for (uint8_t* p : {a, b, c}) {
      B2_TRY(ntt_run(ctx, p, z.log_n, B200ZK_NTT_INVERSE, nullptr, st));
      B2_TRY(ntt_run(ctx, p, z.log_n, B200ZK_NTT_COSET, z.omega, st));
    }
    B2_TRY(fr_quotient_dev(ctx, a, b, c, a, n, (const uint32_t*)z.one.p, st));
  }
  // ---- the MSMs (H over P as Montgomery scalars, all domainSize points), then the key terms and the blinding
  b200zk_groth16_pk pk{};
  pk.log_n = z.log_n;
  const uint64_t counts[5] = {nv, nv, nv, nv - z.n_public - 1, n}, offsets[5] = {0, 0, 0, (uint64_t)z.n_public + 1, 0};
  for (int k = 0; k < 5; ++k) { pk.handle[k] = z.col[k]; pk.count[k] = counts[k]; pk.offset[k] = offsets[k]; }
  B2_TRY(groth16_commit_partials(ctx, &pk, wit, a, nullptr, nullptr, B200ZK_G16_INPUTS_DEVICE | B200ZK_G16_H_COEFFS, st, ctx->ws_g16[3].p));
  B2_TRY(groth16_assemble_zk_dev(ctx, ctx->ws_g16[3].p, 1, g1, g2, zk.r, zk.s, st, ctx->ws_out.p));
  B2_CUDA(ctx, cudaMemcpyAsync(ctx->h_pinned, ctx->ws_out.p, 256, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(ctx->h_pinned + 256, bad, 8, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  unsigned long long first_bad;
  memcpy(&first_bad, ctx->h_pinned + 256, 8);
  if (first_bad != ~0ull) {
    char msg[128];
    snprintf(msg, sizeof msg, "wtns: section 2: value %llu is >= r", first_bad);
    return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, msg);
  }
  memcpy(proof, ctx->h_pinned, 256);
  return B200ZK_OK;
}

}  // namespace
}  // namespace b200zk

using namespace b200zk;

extern "C" {

int b200zk_groth16_zkey_load(b200zk_ctx* ctx, const void* zkey, size_t len, int precompute, uint64_t* key) {
  if (!ctx || !key) return fail(ctx, B200ZK_ERR_INVALID_ARG, "zkey_load: null argument");
  DeviceGuard guard(ctx);
  return load(ctx, (const uint8_t*)zkey, len, precompute, key);
}

int b200zk_groth16_zkey_free(b200zk_ctx* ctx, uint64_t key) {
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  DeviceGuard guard(ctx);
  ZkeyEntry* z = find_zkey(ctx, key, "zkey_free: unknown key");
  if (!z) return B200ZK_ERR_INVALID_ARG;
  B2_CUDA(ctx, cudaDeviceSynchronize());
  for (uint64_t h : z->col) ctx->bases.erase(h);
  ctx->bases.erase(z->terms_g1);
  ctx->bases.erase(z->terms_g2);
  ctx->zkeys.erase(key);
  return B200ZK_OK;
}

int b200zk_groth16_zkey_info(b200zk_ctx* ctx, uint64_t key, uint32_t* n_vars, uint32_t* n_public, uint32_t* log_n, uint8_t* vk, size_t vk_len) {
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  const ZkeyEntry* z = find_zkey(ctx, key, "zkey_info: unknown key");
  if (!z) return B200ZK_ERR_INVALID_ARG;
  if (n_vars) *n_vars = z->n_vars;
  if (n_public) *n_public = z->n_public;
  if (log_n) *log_n = z->log_n;
  if (vk) {
    if (vk_len < z->vk.size()) return fail(ctx, B200ZK_ERR_INVALID_ARG, "zkey_info: vk buffer shorter than 448 + 64 (nPublic + 1) bytes");
    memcpy(vk, z->vk.data(), z->vk.size());
  }
  return B200ZK_OK;
}

int b200zk_groth16_zkey_prove(b200zk_ctx* ctx, uint64_t key, const void* wtns, size_t len, const uint8_t r[32], const uint8_t s[32], void* stream,
                              uint8_t proof[256]) {
  if (!ctx || !r || !s || !proof) return fail(ctx, B200ZK_ERR_INVALID_ARG, "zkey_prove: null argument");
  DeviceGuard guard(ctx);
  const ZkeyEntry* z = find_zkey(ctx, key, "zkey_prove: unknown key");
  if (!z) return B200ZK_ERR_INVALID_ARG;
  return prove(ctx, *z, (const uint8_t*)wtns, len, r, s, pick_stream(ctx, stream), proof);
}

}  // extern "C"
