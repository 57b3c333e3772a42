// ntt.cu -- number-theoretic transform over the BN254 scalar field Fr for sm_90a.
//
// Replaces ark_poly::Radix2EvaluationDomain::{fft,ifft,coset_fft,coset_ifft}_in_place (ark-poly 0.5.0,
// /root/reference/Cargo.lock:1140; equal to gnark-crypto bn254 fr/fft) as used by the Groth16 wrap behind
// /root/reference/crates/prover/src/backend/sp1.rs:97-134 (SURVEY.md section 8a row a8).
//   out[k] = sum_j a[j] * w^(jk),  natural order in and out,  w = g^(2^(28-log_n)),  g = 5^((r-1)/2^28).
//
// Schedule: merged-stage Cooley-Tukey in Stockham (auto-sort) form.  log_n stages are split into P passes
// of s_p stages; pass p with Ns = prod_{q<p} 2^(s_q) and R = 2^(s_p) computes, for every j in [0, N/R):
//     v[r]  = in[j + r*N/R] * w_N^( r * (j mod Ns) * N/(Ns*R) )          (inter-pass twiddle)
//     V     = NTT_R(v)                                                     (s_p radix-2 stages in shared memory)
//     out[(j div Ns)*Ns*R + (j mod Ns) + q*Ns] = V[q]
// One CTA owns a tile of 2^t adjacent j, so every global access is a run of 2^t * 32 B, and the R-point
// transforms of a tile never leave shared memory.  Inter-pass twiddles come from one 2^16-entry table when
// Ns*R <= 2^16 (a single lookup); the LAST pass of a larger transform streams them from a direct N-entry table
// (NttTables::full: the pass is bound by products, not by HBM, and one lookup costs one product instead of two);
// any other pass, and sizes beyond the table's cap, use two 4096-entry tables (w^lo, w^(hi*4096)) and one extra product.
#include "common.cuh"
#include "tma.cuh"
#include <cstdlib>
#include <cstring>

namespace b200zk {

static constexpr int kLoBits = 12;
static constexpr int kMaxStage = 12;  // 2^12 elements * 32 B = 128 KiB of shared memory

// device table layout (in Fr elements)
struct NttTables {
  const uint4* stage;  // stage[(2^(s-1) - 1) + i] = w_{2^s}^i, s = 1..12
  const uint4* lo;     // lo[x] = w_N^x, x < 2^min(12, k)
  const uint4* hi;     // hi[y] = w_N^(y << 12)
  const uint4* ninv;   // n^-1
  const uint4* d16;    // d16[x] = w_{2^16}^x, x < 2^16: inter-pass twiddles of passes with Ns*R <= 2^16 in ONE lookup
  const uint4* lo_n;   // lo_n[x] = lo[x] * n^-1: the last pass of an inverse transform scales through its twiddles
  const uint4* full;   // last pass with Ns*R = N > 2^16 only, or nullptr: full[(r << log_ns) + jm] = w_N^(r*jm) (* n^-1 when the
                       // pass folds the scale): ONE streamed lookup and one product per element instead of two lookups and
                       // two products -- HBM has the room (N * 32 B per table) and the pass the bandwidth (it is product bound)
};
static constexpr uint32_t kDirectBits = 16;

// The 2^28-th primitive root of unity the domain generators derive from is a PARAMETER (SURVEY.md section 8c): the
// context default is ark-poly / gnark-crypto's 5^((r-1)/2^28) = 0x2a3c09f0a58a7e85...725b19f0; halo2curves (the
// OpenVM wrap, /root/reference/crates/prover/src/backend/openvm.rs:52-56) uses 7^((r-1)/2^28) = 0x03ddb9f5...60c37c9c.
struct RootArg { uint32_t v[8]; };  // canonical limbs
B2_D Fr fr_root_2_28(const RootArg& g) {
  Fr c;
#pragma unroll
  for (int i = 0; i < 8; ++i) c.v[i] = g.v[i];
  return Fr::to_mont(c);
}
B2_D Fr fr_pow_u32(Fr b, uint32_t e) {
  Fr acc = Fr::one();
  while (e) { if (e & 1) acc = Fr::mul(acc, b); b = Fr::sqr(b); e >>= 1; }
  return acc;
}
B2_D Fr root_of_unity(uint32_t log_n, const RootArg& g) {
  Fr w = fr_root_2_28(g);
  for (uint32_t i = log_n; i < 28; ++i) w = Fr::sqr(w);
  return w;
}

// entries: [0, 4095) stage tables, then 2^lb lo, then 2^(k-lb) hi, then n^-1, then 2^16 direct, then 2^lb lo * n^-1
__global__ void __launch_bounds__(128) ntt_build_tables(uint32_t log_n, int inverse, void* out, uint32_t n_lo, uint32_t n_hi, RootArg g) {
  uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t n_stage = (1u << kMaxStage) - 1;
  uint32_t total = n_stage + n_lo + n_hi + 1;
  if (id >= total + (1u << kDirectBits) + n_lo) return;
  Fr val;
  if (id >= total + (1u << kDirectBits)) {
    uint32_t e = id - total - (1u << kDirectBits), N = 1u << log_n;
    if (inverse) e = (N - e) & (N - 1);
    Fr n = Fr::zero(); n.v[0] = N;
    val = fr_pow_u32(root_of_unity(log_n, g), e);
    if (inverse) val = Fr::mul(val, Fr::inv(Fr::to_mont(n)));
    store_fe<Fr>(out, id, val);
    return;
  }
  if (id >= total) {
    uint32_t x = id - total, D = 1u << kDirectBits;
    val = fr_pow_u32(root_of_unity(kDirectBits, g), inverse ? (D - x) & (D - 1) : x);
    store_fe<Fr>(out, id, val);
    return;
  }
  if (id < n_stage) {
    uint32_t s = 32 - __clz(id + 1);           // id+1 in [2^(s-1), 2^s)
    uint32_t i = id + 1 - (1u << (s - 1));
    Fr w = root_of_unity(s, g);
    uint32_t e = inverse ? ((1u << s) - i) & ((1u << s) - 1) : i;
    val = fr_pow_u32(w, e);
  } else if (id < n_stage + n_lo + n_hi) {
    uint32_t x = id - n_stage;
    uint32_t e = x < n_lo ? x : (x - n_lo) << kLoBits;
    uint32_t N = 1u << log_n;  // log_n <= 28
    if (inverse) e = (N - e) & (N - 1);
    val = fr_pow_u32(root_of_unity(log_n, g), e);
  } else {
    Fr n = Fr::zero(); n.v[0] = 1u << log_n;
    val = inverse ? Fr::inv(Fr::to_mont(n)) : Fr::one();
  }
  store_fe<Fr>(out, id, val);
}

// full[(r << lns) + jm] = w_N^(r * jm) for r < 2^(k - lns), jm < 2^lns, from the two-level tables (lo_sel = lo or lo * n^-1)
__global__ void __launch_bounds__(256) ntt_build_full(uint32_t k, uint32_t lns, const uint4* lo_sel, const uint4* hi, void* out) {
  const size_t n = (size_t)1 << k;
  for (size_t id = blockIdx.x * (size_t)blockDim.x + threadIdx.x; id < n; id += (size_t)gridDim.x * blockDim.x) {
    const uint32_t r = (uint32_t)(id >> lns), jm = (uint32_t)id & ((1u << lns) - 1);
    const uint32_t e = r * jm;  // < 2^k
    store_fe<Fr>(out, id, Fr::mul(load_fe_nc<Fr>(lo_sel, e & ((1u << kLoBits) - 1)), load_fe_nc<Fr>(hi, e >> kLoBits)));
  }
}

// flags[0] = 1 iff g^(2^28) == 1 and g^(2^27) != 1 (g canonical, < r)
__global__ void ntt_check_root(RootArg g, uint32_t* flags) {
  if (blockIdx.x || threadIdx.x) return;
  Fr c, m = Fr::modulus(), t;
#pragma unroll
  for (int i = 0; i < 8; ++i) c.v[i] = g.v[i];
  const bool in_range = detail::sub8(t.v, c.v, m.v) != 0;
  Fr w = Fr::to_mont(c);
  for (int i = 0; i < 27; ++i) w = Fr::sqr(w);
  const bool half_is_one = (w == Fr::one());
  w = Fr::sqr(w);
  flags[0] = (in_range && !half_is_one && w == Fr::one()) ? 1u : 0u;
}

struct PassArgs {
  const void* in;
  void* out;
  uint32_t log_n, s, t, log_ns;
  uint32_t scale_out;  // multiply outputs by n^-1
  uint32_t scale_in;   // last pass of an inverse transform: n^-1 rides on the inter-pass twiddles (lo_n), no extra product
  uint32_t coset_in;   // first pass of a forward coset transform: element i enters multiplied by h^i
  uint32_t coset_out;  // last pass of an inverse coset transform: element i leaves multiplied by h^-i * n^-1
  const uint4* c_lo;   // coset powers, low table  (base^x, x < 4096; the inverse one carries n^-1)
  const uint4* c_hi;   // coset powers, high table (base^(y << 12))
  NttTables tb;
};

// v * base^i from the two-level coset tables
B2_D Fr coset_scale(const Fr& v, size_t i, uint32_t k, const uint4* lo, const uint4* hi) {
  Fr tw = load_fe_nc<Fr>(lo, i & ((1u << kLoBits) - 1));
  if (k > (uint32_t)kLoBits) tw = Fr::mul(tw, load_fe_nc<Fr>(hi, i >> kLoBits));
  return Fr::mul(v, tw);
}

B2_D Fr lds_fr(const uint4* sm, uint32_t i) {
  uint4 lo = sm[2 * i], hi = sm[2 * i + 1];
  Fr r;
  r.v[0] = lo.x; r.v[1] = lo.y; r.v[2] = lo.z; r.v[3] = lo.w; r.v[4] = hi.x; r.v[5] = hi.y; r.v[6] = hi.z; r.v[7] = hi.w;
  return r;
}
B2_D void sts_fr(uint4* sm, uint32_t i, const Fr& a) {
  sm[2 * i] = make_uint4(a.v[0], a.v[1], a.v[2], a.v[3]);
  sm[2 * i + 1] = make_uint4(a.v[4], a.v[5], a.v[6], a.v[7]);
}

// v * w_{2^L}^(r*jm): one lookup when L <= 16, else two lookups and a product
B2_D Fr interpass_twiddle(const Fr& v, uint32_t r, uint32_t jm, uint32_t k, uint32_t lns, uint32_t L, const NttTables& tb, bool scaled) {
  const uint32_t x = r * jm;
  if (!x) return scaled ? Fr::mul(v, load_fe_nc<Fr>(tb.ninv, 0)) : v;
  Fr tw;
  if (tb.full) {           // only set for the pass it was built for (L == k)
    tw = load_fe_nc<Fr>(tb.full, ((size_t)r << lns) + jm);
  } else if (L <= kDirectBits) {  // scaled is only requested for L > 16
    tw = load_fe_nc<Fr>(tb.d16, x << (kDirectBits - L));
  } else {
    uint32_t e = x << (k - L);
    tw = Fr::mul(load_fe_nc<Fr>(scaled ? tb.lo_n : tb.lo, e & ((1u << kLoBits) - 1)), load_fe_nc<Fr>(tb.hi, e >> kLoBits));
  }
  return Fr::mul(v, tw);
}

template <int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB) ntt_pass(PassArgs a) {
  extern __shared__ uint4 sm[];
  const uint32_t k = a.log_n, s = a.s, t = a.t, lns = a.log_ns;
  const uint32_t R = 1u << s, cols = 1u << t, cmask = cols - 1;
  const uint32_t ns_mask = (1u << lns) - 1;
  const uint32_t stride_log = k - s;                         // N/R
  const uint32_t j0 = blockIdx.x << t;
  const uint32_t items = R << t;

  // ---- load: the tile is R rows of 2^t * 32 contiguous bytes (one run when the tile is the whole input); the
  // copy engine (cp.async.bulk, mbarrier completion) lands them in shared memory as sm[(r << t) + c]
  __shared__ uint64_t tile_bar;
  if (threadIdx.x == 0) { tma::barrier_init(&tile_bar, 1); tma::barrier_init_fence(); }
  __syncthreads();
  {
    const uint8_t* src = reinterpret_cast<const uint8_t*>(a.in);
    if (threadIdx.x == 0) tma::barrier_expect(&tile_bar, items * 32u);
    if (stride_log == t) {  // rows are adjacent in memory: one bulk copy
      if (threadIdx.x == 0) tma::bulk_load(sm, src + (size_t)j0 * 32, items * 32u, &tile_bar);
    } else {
      for (uint32_t r = threadIdx.x; r < R; r += THREADS)
        tma::bulk_load(sm + 2 * ((size_t)r << t), src + ((size_t)j0 + ((size_t)r << stride_log)) * 32, cols * 32u, &tile_bar);
    }
    // while the tile is in flight: pull this tile's slice of the direct twiddle table (R runs of 2^t * 32 B) into L2,
    // so that the first round's lookups do not pay HBM latency on top of the tile's
    if (lns && a.tb.full) {
      const uint8_t* tw = reinterpret_cast<const uint8_t*>(a.tb.full);
      for (uint32_t r = threadIdx.x; r < R; r += THREADS) {
        const uint8_t* p = tw + ((((size_t)r << lns) + (j0 & ns_mask)) << 5);
        for (uint32_t b = 0; b < cols * 32u; b += 128) asm volatile("prefetch.global.L2 [%0];" ::"l"(p + b));
      }
    }
    tma::barrier_wait(&tile_bar, 0);
  }

  // ---- s decimation-in-frequency stages in shared memory, two stages per round trip (radix-4 in registers):
  // a thread holds rows {i, i+m/2, i+m, i+3m/2}, does the stage-q butterflies (i,i+m), (i+m/2,i+3m/2) and then
  // the stage-(q+1) butterflies (i,i+m/2), (i+m,i+3m/2) before anything goes back to shared memory -- half the
  // LDS/STS traffic and half the barriers of a stage-by-stage sweep.  An odd s starts with one radix-2 stage.
  const uint4* stage_tw = a.tb.stage + 2 * ((size_t)(R >> 1) - 1);
  auto first_touch = [&](Fr v, uint32_t row, uint32_t c) -> Fr {
    if (a.coset_in) v = coset_scale(v, (size_t)(j0 + c) + ((size_t)row << stride_log), k, a.c_lo, a.c_hi);  // h^index
    if (lns) v = interpass_twiddle(v, row, (j0 + c) & ns_mask, k, lns, lns + s, a.tb, a.scale_in != 0);  // w_{2^L}^(row * (j mod Ns))
    return v;
  };
  uint32_t q = 0;
  if (s & 1) {
    const uint32_t lm = s - 1, m = 1u << lm;
    for (uint32_t it = threadIdx.x; it < (items >> 1); it += THREADS) {
      uint32_t c = it & cmask, jj = it >> t;  // one block: blk = 0
      uint32_t p0 = (jj << t) + c, p1 = ((jj + m) << t) + c;
      Fr x = first_touch(lds_fr(sm, p0), jj, c), y = first_touch(lds_fr(sm, p1), jj + m, c);
      Fr d = Fr::sub(x, y);
      if (jj) d = Fr::mul(d, load_fe_nc<Fr>(stage_tw, jj));
      sts_fr(sm, p0, Fr::add(x, y));
      sts_fr(sm, p1, d);
    }
    __syncthreads();
    q = 1;
  }
  for (; q < s; q += 2) {
    const uint32_t lm = s - 1 - q, m = 1u << lm, m2 = m >> 1;
    // quad u = (block, jj), jj < m/2.  With jj in the HIGH bits of u the lanes of a warp share one jj: twiddle
    // loads are broadcasts and the jj == 0 quads (w^0 = 1 on three of their four products) skip them warp-uniformly.
    const uint32_t nblk_log = q;             // R / (2m) blocks
    const bool uniform = nblk_log >= 2;
    for (uint32_t it = threadIdx.x; it < (items >> 2); it += THREADS) {
      uint32_t c = it & cmask, u = it >> t;
      uint32_t jj = uniform ? (u >> nblk_log) : (u & (m2 - 1));
      uint32_t blk = uniform ? (u & ((1u << nblk_log) - 1)) : (u >> (lm - 1));
      uint32_t i = (blk << (lm + 1)) | jj;
      uint32_t pa = (i << t) + c, pb = ((i + m2) << t) + c, pc = ((i + m) << t) + c, pd = ((i + m + m2) << t) + c;
      Fr A = lds_fr(sm, pa), B = lds_fr(sm, pb), C = lds_fr(sm, pc), D = lds_fr(sm, pd);
      if (q == 0) { A = first_touch(A, i, c); B = first_touch(B, i + m2, c); C = first_touch(C, i + m, c); D = first_touch(D, i + m + m2, c); }
      // stage q: distance m, twiddles w_{2m}^jj and w_{2m}^(jj + m/2)
      Fr t0 = Fr::add(A, C), t1 = Fr::sub(A, C), t2 = Fr::add(B, D), t3 = Fr::sub(B, D);
      if (jj) t1 = Fr::mul(t1, load_fe_nc<Fr>(stage_tw, jj << q));
      t3 = Fr::mul(t3, load_fe_nc<Fr>(stage_tw, (jj + m2) << q));
      // stage q+1: distance m/2, twiddle w_m^jj for both butterflies
      Fr o0 = Fr::add(t0, t2), o1 = Fr::sub(t0, t2), o2 = Fr::add(t1, t3), o3 = Fr::sub(t1, t3);
      if (jj) {
        Fr w = load_fe_nc<Fr>(stage_tw, jj << (q + 1));
        o1 = Fr::mul(o1, w); o3 = Fr::mul(o3, w);
      }
      sts_fr(sm, pa, o0); sts_fr(sm, pb, o1); sts_fr(sm, pc, o2); sts_fr(sm, pd, o3);
    }
    __syncthreads();
  }

  // ---- store: V[q] sits at bit-reversed row brev_s(q)
  const Fr ninv = a.scale_out ? load_fe_nc<Fr>(a.tb.ninv, 0) : Fr::one();
  if (lns == 0) {
    // first pass: out[j*R + q], q fastest => the tile is one contiguous run of R * 2^t elements
    for (uint32_t it = threadIdx.x; it < items; it += THREADS) {
      uint32_t q = it & (R - 1), c = it >> s;
      uint32_t row = s ? (__brev(q) >> (32 - s)) : 0;
      Fr v = lds_fr(sm, (row << t) + c);
      const size_t o = (((size_t)(j0 + c)) << s) + q;
      if (a.scale_out) v = Fr::mul(v, ninv);
      if (a.coset_out) v = coset_scale(v, o, k, a.c_lo, a.c_hi);
      store_fe<Fr>(a.out, o, v);
    }
  } else {
    for (uint32_t it = threadIdx.x; it < items; it += THREADS) {
      uint32_t c = it & cmask, q = it >> t;
      uint32_t row = s ? (__brev(q) >> (32 - s)) : 0;
      uint32_t j = j0 + c;
      Fr v = lds_fr(sm, (row << t) + c);
      if (a.scale_out) v = Fr::mul(v, ninv);
      size_t o = (((size_t)(j >> lns)) << (lns + s)) + (j & ns_mask) + ((size_t)q << lns);
      if (a.coset_out) v = coset_scale(v, o, k, a.c_lo, a.c_hi);
      store_fe<Fr>(a.out, o, v);
    }
  }
}

// data[i] *= hi[i >> 12] * lo[i & 4095]   (coset shift h^i, or h^-i * n^-1)
__global__ void __launch_bounds__(256) ntt_scale_pow(void* data, size_t n, const void* lo, const void* hi, int has_hi) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    Fr tw = load_fe_nc<Fr>(lo, i & ((1u << kLoBits) - 1));
    if (has_hi) tw = Fr::mul(tw, load_fe_nc<Fr>(hi, i >> kLoBits));
    store_fe<Fr>(data, i, Fr::mul(load_fe<Fr>(data, i), tw));
  }
}
// lo[x] = base^x * scale (x < n_lo), hi[y] = base^(y << 12) (y < n_hi); base given canonical
__global__ void __launch_bounds__(128) ntt_build_pow_tables(const uint32_t* base_canonical, int invert, int scale_ninv, uint32_t log_n, void* lo, uint32_t n_lo, void* hi, uint32_t n_hi) {
  uint32_t id = blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= n_lo + n_hi) return;
  Fr b;
#pragma unroll
  for (int i = 0; i < 8; ++i) b.v[i] = base_canonical[i];
  b = Fr::to_mont(b);
  if (invert) b = Fr::inv(b);
  if (id < n_lo) {
    Fr v = fr_pow_u32(b, id);
    if (scale_ninv) { Fr n = Fr::zero(); n.v[0] = 1u << log_n; v = Fr::mul(v, Fr::inv(Fr::to_mont(n))); }
    store_fe<Fr>(lo, id, v);
  } else {
    store_fe<Fr>(hi, id - n_lo, fr_pow_u32(b, (id - n_lo) << kLoBits));
  }
}

// canonical <-> Montgomery (+ optional byte order), in place
__global__ void __launch_bounds__(256) fr_convert(void* data, size_t n, int to_mont, int big_endian) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    Fr v = load_fe<Fr>(data, i);
    if (to_mont) {
      if (big_endian) { Fr w; for (int k = 0; k < 8; ++k) w.v[k] = __byte_perm(v.v[7 - k], 0, 0x0123); v = w; }
      for (int k = 0; k < 5; ++k) { Fr m = Fr::modulus(), tt; if (!detail::sub8(tt.v, v.v, m.v)) v = tt; }
      v = Fr::to_mont(v);
    } else {
      v = Fr::from_mont(v);
      if (big_endian) { Fr w; for (int k = 0; k < 8; ++k) w.v[k] = __byte_perm(v.v[7 - k], 0, 0x0123); v = w; }
    }
    store_fe<Fr>(data, i, v);
  }
}

// ---- host side ----------------------------------------------------------------------------------------------
static int get_tables(b200zk_ctx* ctx, uint32_t log_n, bool inverse, cudaStream_t st, NttTables* out) {
  const uint64_t key = ((uint64_t)log_n | ((uint64_t)inverse << 8)) ^ (ctx->ntt_root_id << 9);  // root id 0 (default) keeps the plain key
  const uint32_t n_stage = (1u << kMaxStage) - 1;
  const uint32_t lb = log_n < (uint32_t)kLoBits ? log_n : (uint32_t)kLoBits;
  const uint32_t n_lo = 1u << lb, n_hi = log_n > (uint32_t)kLoBits ? 1u << (log_n - kLoBits) : 1u;
  auto it = ctx->twiddles.find(key);
  if (it == ctx->twiddles.end()) {
    TwiddleSet ts;
    ts.bytes = (size_t)(n_stage + n_lo + n_hi + 1 + (1u << kDirectBits) + n_lo) * 32;
    B2_CUDA(ctx, cudaMalloc(&ts.d, ts.bytes));
    uint32_t total = n_stage + n_lo + n_hi + 1 + (1u << kDirectBits) + n_lo;
    RootArg g;
    memcpy(g.v, ctx->ntt_root, 32);
    memcpy(ts.root, ctx->ntt_root, 32);
    B2_LAUNCH(ctx, ntt_build_tables, (total + 127) / 128, 128, 0, st, log_n, inverse ? 1 : 0, ts.d, n_lo, n_hi, g);
    // a later transform of this size on ANOTHER stream must not read half-built tables
    if (cudaEventCreateWithFlags(&ts.ready, cudaEventDisableTiming) == cudaSuccess) cudaEventRecord(ts.ready, st); else { cudaGetLastError(); ts.ready = nullptr; B2_CUDA(ctx, cudaStreamSynchronize(st)); }
    it = ctx->twiddles.emplace(key, ts).first;
  } else if (memcmp(it->second.root, ctx->ntt_root, 32) != 0) {
    return fail(ctx, B200ZK_ERR_CUDA, "ntt: twiddle cache key collision between two roots of unity");
  }
  if (it->second.ready) B2_CUDA(ctx, cudaStreamWaitEvent(st, it->second.ready, 0));
  const uint4* base = (const uint4*)it->second.d;
  out->stage = base;
  out->lo = base + 2 * (size_t)n_stage;
  out->hi = out->lo + 2 * (size_t)n_lo;
  out->ninv = out->hi + 2 * (size_t)n_hi;
  out->d16 = out->ninv + 2;
  out->lo_n = out->d16 + 2 * ((size_t)1 << kDirectBits);
  out->full = nullptr;
  return B200ZK_OK;
}

// The last pass's direct twiddle table (NttTables::full), built on first use per (size, direction, root, last-pass width,
// scaled).  Largest size: B200ZK_NTT_FULL_TW (default 26 -> 2 GiB per table; 0 disables).  Any failure to allocate leaves
// *out = nullptr and the pass on the two-level tables: this is an optimisation, never a requirement.
static int get_full_table(b200zk_ctx* ctx, uint32_t log_n, bool inverse, uint32_t s_last, bool scaled, const NttTables& tb, cudaStream_t st, const uint4** out) {
  *out = nullptr;
  const char* knob = getenv("B200ZK_NTT_FULL_TW");  // read per call: tests switch it inside one process
  const int max_log = (knob && *knob) ? atoi(knob) : 26;
  if (log_n <= kDirectBits || (int)log_n > max_log || s_last >= log_n) return B200ZK_OK;
  uint32_t tag[8] = {0xF0117ab1u, log_n, inverse ? 1u : 0u, s_last, scaled ? 1u : 0u, 0, 0, 0};
  uint64_t key = 0xcbf29ce484222325ull ^ ctx->ntt_root_id;
  for (int i = 0; i < 5; ++i) key = (key ^ tag[i]) * 0x100000001b3ull;
  key |= 1ull << 63;
  auto it = ctx->twiddles.find(key);
  if (it != ctx->twiddles.end() && (memcmp(it->second.gen, tag, 32) != 0 || memcmp(it->second.root, ctx->ntt_root, 32) != 0)) return B200ZK_OK;  // key collision: do without
  if (it == ctx->twiddles.end()) {
    TwiddleSet ts;
    memcpy(ts.gen, tag, 32);
    memcpy(ts.root, ctx->ntt_root, 32);
    ts.bytes = ((size_t)1 << log_n) * 32;
    if (cudaMalloc(&ts.d, ts.bytes) != cudaSuccess) { cudaGetLastError(); return B200ZK_OK; }
    B2_LAUNCH(ctx, ntt_build_full, ctx->sm_count * 8, 256, 0, st, log_n, log_n - s_last, scaled ? tb.lo_n : tb.lo, tb.hi, ts.d);
    if (cudaEventCreateWithFlags(&ts.ready, cudaEventDisableTiming) == cudaSuccess) cudaEventRecord(ts.ready, st); else { cudaGetLastError(); ts.ready = nullptr; B2_CUDA(ctx, cudaStreamSynchronize(st)); }
    it = ctx->twiddles.emplace(key, ts).first;
  }
  if (it->second.ready) B2_CUDA(ctx, cudaStreamWaitEvent(st, it->second.ready, 0));
  *out = (const uint4*)it->second.d;
  return B200ZK_OK;
}

struct Plan { int P; uint32_t s[4]; uint32_t t[4]; };

static Plan make_ntt_plan(uint32_t k) {
  Plan p{};
  if (k <= (uint32_t)kMaxStage) { p.P = 1; p.s[0] = k; }
  // 64 KiB tiles keep several CTAs per SM to cover barrier and copy latency, so stages are capped at 10-11
  else if (k <= 20) { p.P = 2; p.s[0] = (k + 1) / 2; p.s[1] = k - p.s[0]; }
  else { p.P = 3; p.s[0] = (k + 2) / 3; p.s[1] = (k - p.s[0] + 1) / 2; p.s[2] = k - p.s[0] - p.s[1]; }
  const uint32_t tile_log = 11;  // 2048 elements = 64 KiB per CTA
  for (int i = 0; i < p.P; ++i) {
    uint32_t tl = tile_log < p.s[i] ? p.s[i] : tile_log;
    p.t[i] = tl - p.s[i];
    uint32_t jbits = k - p.s[i];  // number of j values = 2^(k-s)
    if (p.t[i] > jbits) p.t[i] = jbits;
  }
  return p;
}

static int launch_pass(b200zk_ctx* ctx, const PassArgs& a, cudaStream_t st) {
  const uint32_t items = 1u << (a.s + a.t);
  const size_t smem = (size_t)items * 32;
  const unsigned grid = 1u << (a.log_n - a.s - a.t);
  if (items >= 4096) {
    // the opt-in to > 48 KiB of dynamic shared memory is a per-device function attribute: remembered per context
    if (!ctx->attr_ntt512) { B2_CUDA(ctx, cudaFuncSetAttribute((ntt_pass<512, 1>), cudaFuncAttributeMaxDynamicSharedMemorySize, 1 << 17)); ctx->attr_ntt512 = true; }
    B2_LAUNCH(ctx, (ntt_pass<512, 1>), grid, 512, smem, st, a);
  } else {
    // 64 KiB tiles: three CTAs fit an SM's shared memory; MINB = 3 caps registers at 85 so that they also fit
    // its register file
    if (!ctx->attr_ntt256) { B2_CUDA(ctx, cudaFuncSetAttribute((ntt_pass<256, 3>), cudaFuncAttributeMaxDynamicSharedMemorySize, 1 << 16)); ctx->attr_ntt256 = true; }
    B2_LAUNCH(ctx, (ntt_pass<256, 3>), grid, 256, smem, st, a);
  }
  return B200ZK_OK;
}

// root_le: canonical little-endian limbs of a primitive 2^28-th root of unity of Fr, or nullptr for the default
int ntt_set_root(b200zk_ctx* ctx, const uint8_t* root_le) {
  static const uint32_t kDefault[8] = {0x725b19f0u, 0x9bd61b6eu, 0x41112ed4u, 0x402d111eu, 0x8ef62abcu, 0x00e0a7ebu, 0xa58a7e85u, 0x2a3c09f0u};
  if (!root_le || memcmp(root_le, kDefault, 32) == 0) { memcpy(ctx->ntt_root, kDefault, 32); ctx->ntt_root_id = 0; return B200ZK_OK; }
  RootArg g;
  memcpy(g.v, root_le, 32);
  B2_TRY(ensure(ctx, ctx->ws_result, 256));
  cudaStream_t st = ctx->stream;
  B2_LAUNCH(ctx, ntt_check_root, 1, 32, 0, st, g, (uint32_t*)ctx->ws_result.p);
  B2_CUDA(ctx, cudaMemcpyAsync(ctx->h_pinned + 3584, ctx->ws_result.p, 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  uint32_t ok; memcpy(&ok, ctx->h_pinned + 3584, 4);
  if (!ok) return fail(ctx, B200ZK_ERR_INVALID_ARG, "ntt root: not a primitive 2^28-th root of unity of Fr");
  memcpy(ctx->ntt_root, g.v, 32);
  uint64_t id = 0xcbf29ce484222325ull;
  for (int i = 0; i < 8; ++i) id = (id ^ g.v[i]) * 0x100000001b3ull;
  ctx->ntt_root_id = (id >> 10) | 1;  // non-zero, fits under the key's tag bit after the << 9
  return B200ZK_OK;
}

int ntt_run(b200zk_ctx* ctx, void* d_data, uint32_t log_n, uint32_t flags, const uint8_t* coset_gen, cudaStream_t st) {
  NvtxRange nvtx_ntt("b200zk:fr_ntt");
  if (log_n > 28) return fail(ctx, B200ZK_ERR_INVALID_ARG, "ntt: log_n > 28 (two-adicity of Fr)");
  if ((uintptr_t)d_data & 15) return fail(ctx, B200ZK_ERR_INVALID_ARG, "ntt: the device buffer must be 16-byte aligned");
  const size_t n = (size_t)1 << log_n;
  const bool inverse = flags & B200ZK_NTT_INVERSE, coset = flags & B200ZK_NTT_COSET;
  const bool canonical = flags & (B200ZK_NTT_CANONICAL | B200ZK_NTT_BE), be = flags & B200ZK_NTT_BE;
  const unsigned egrid = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 32);
  if (canonical) B2_LAUNCH(ctx, fr_convert, egrid, 256, 0, st, d_data, n, 1, be ? 1 : 0);

  void *c_lo = nullptr, *c_hi = nullptr;
  const uint32_t lb = log_n < (uint32_t)kLoBits ? log_n : (uint32_t)kLoBits;
  const uint32_t n_lo = 1u << lb, n_hi = log_n > (uint32_t)kLoBits ? 1u << (log_n - kLoBits) : 1u;
  if (coset) {
    uint32_t h[8] = {5, 0, 0, 0, 0, 0, 0, 0};
    if (coset_gen) {
      if (be) for (int i = 0; i < 8; ++i) h[i] = ((uint32_t)coset_gen[31 - 4 * i]) | ((uint32_t)coset_gen[30 - 4 * i] << 8) | ((uint32_t)coset_gen[29 - 4 * i] << 16) | ((uint32_t)coset_gen[28 - 4 * i] << 24);
      else memcpy(h, coset_gen, 32);
    }
    // tables of h^i (or h^-i * n^-1) are cached per (log_n, direction, generator): a prover uses one generator,
    // and the inverse table costs two serial field inversions to build
    uint64_t key = 0xcbf29ce484222325ull ^ ((uint64_t)log_n | ((uint64_t)inverse << 8) | (1ull << 16));
    for (int i = 0; i < 8; ++i) key = (key ^ h[i]) * 0x100000001b3ull;
    key |= 1ull << 63;  // never collides with the twiddle keys (log_n | inverse << 8)
    auto it = ctx->twiddles.find(key);
    if (it != ctx->twiddles.end() && memcmp(it->second.gen, h, 32) != 0) {  // 64-bit key collision: rebuild
      B2_CUDA(ctx, cudaDeviceSynchronize());
      cudaFree(it->second.d);
      if (it->second.ready) cudaEventDestroy(it->second.ready);
      ctx->twiddles.erase(it);
      it = ctx->twiddles.end();
    }
    if (it == ctx->twiddles.end()) {
      TwiddleSet ts;
      memcpy(ts.gen, h, 32);
      ts.bytes = (size_t)(n_lo + n_hi) * 32 + 64;
      B2_CUDA(ctx, cudaMalloc(&ts.d, ts.bytes));
      B2_CUDA(ctx, cudaMemcpyAsync(ts.d, h, 32, cudaMemcpyHostToDevice, st));
      B2_CUDA(ctx, cudaStreamSynchronize(st));  // h is a stack buffer
      uint8_t* base = (uint8_t*)ts.d;
      B2_LAUNCH(ctx, ntt_build_pow_tables, (n_lo + n_hi + 127) / 128, 128, 0, st, (const uint32_t*)base, inverse ? 1 : 0, inverse ? 1 : 0, log_n,
                (void*)(base + 64), n_lo, (void*)(base + 64 + (size_t)n_lo * 32), n_hi);
      if (cudaEventCreateWithFlags(&ts.ready, cudaEventDisableTiming) == cudaSuccess) cudaEventRecord(ts.ready, st); else { cudaGetLastError(); ts.ready = nullptr; B2_CUDA(ctx, cudaStreamSynchronize(st)); }
      it = ctx->twiddles.emplace(key, ts).first;
    }
    if (it->second.ready) B2_CUDA(ctx, cudaStreamWaitEvent(st, it->second.ready, 0));
    uint8_t* base = (uint8_t*)it->second.d;
    c_lo = base + 64; c_hi = base + 64 + (size_t)n_lo * 32;
    // log_n == 0 has no pass to fuse into: scale the single element directly
    if (!inverse && log_n == 0) B2_LAUNCH(ctx, ntt_scale_pow, egrid, 256, 0, st, d_data, n, c_lo, c_hi, 0);
  }

  if (log_n > 0) {
    NttTables tb;
    B2_TRY(get_tables(ctx, log_n, inverse, st, &tb));
    Plan pl = make_ntt_plan(log_n);
    if (pl.P > 1) B2_TRY(ensure(ctx, ctx->ws_ntt, n * 32));
    void* bufs[2] = {d_data, ctx->ws_ntt.p};
    uint32_t log_ns = 0;
    int cur = 0;
    for (int p = 0; p < pl.P; ++p) {
      PassArgs a;
      // the last pass reads and writes the same index set per CTA (j + r * 2^(k-s)), after a barrier: it may run in
      // place, which lands an odd number of passes back in the caller's buffer without a trailing copy
      const bool last = p == pl.P - 1, in_place = pl.P == 1 || (last && (pl.P & 1));
      a.in = bufs[cur];
      a.out = in_place ? bufs[cur] : bufs[cur ^ 1];
      a.log_n = log_n; a.s = pl.s[p]; a.t = pl.t[p]; a.log_ns = log_ns;
      const bool fold = inverse && !coset && last && log_ns > 0 && log_n > kDirectBits;
      a.scale_in = fold ? 1 : 0;
      a.scale_out = (inverse && !coset && last && !fold) ? 1 : 0;
      a.coset_in = (coset && !inverse && p == 0) ? 1 : 0;
      a.coset_out = (coset && inverse && p == pl.P - 1) ? 1 : 0;
      a.c_lo = (const uint4*)c_lo; a.c_hi = (const uint4*)c_hi;
      a.tb = tb;
      if (last && log_ns > 0) B2_TRY(get_full_table(ctx, log_n, inverse, pl.s[p], fold, tb, st, &a.tb.full));
      B2_TRY(launch_pass(ctx, a, st));
      log_ns += pl.s[p];
      if (!in_place) cur ^= 1;
    }
    if (pl.P > 1 && cur == 1) B2_CUDA(ctx, cudaMemcpyAsync(d_data, ctx->ws_ntt.p, n * 32, cudaMemcpyDeviceToDevice, st));
  }
  if (coset && inverse && log_n == 0) B2_LAUNCH(ctx, ntt_scale_pow, egrid, 256, 0, st, d_data, n, c_lo, c_hi, 0);
  if (canonical) B2_LAUNCH(ctx, fr_convert, egrid, 256, 0, st, d_data, n, 0, be ? 1 : 0);
  return B200ZK_OK;
}

}  // namespace b200zk
