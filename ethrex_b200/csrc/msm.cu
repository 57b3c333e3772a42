// msm.cu -- windowed Pippenger multi-scalar multiplication over BN254 G1 / G2 for sm_90a.
//
// Replaces ark_ec::VariableBaseMSM::msm (ark-ec 0.5.0, /root/reference/Cargo.lock:978) as reached by the
// Groth16 wrap behind /root/reference/crates/prover/src/backend/sp1.rs:97-134 and risc0.rs:24-29,71-82
// (SURVEY.md section 8a rows a6/a7).  Same digit rule as ark's `make_digits` (signed radix-2^c digits, carry
// when the window value >= 2^(c-1), 2^(c-1) buckets per window), but the schedule is GPU shaped (msm_run):
//
//   1. digit sort    recode every scalar into W signed digits and sort the (window,bucket) entries: each becomes a
//                    point index with the digit's sign in bit 31, bucket-major.  The two-level sort (msm_sort_*: tile-
//                    local counting sorts in shared memory) from 2^16 points up; below that the one-pass sort (msm_hist
//                    histogram, scan, msm_scatter);
//   2. scan_*        exclusive prefix sums -> the runs' offsets (3 small kernels, exclusive_scan);
//   3. msm_accumulate  THE hot kernel: one thread per fixed SLICE of <= 256 sorted entries (perfectly balanced):
//                    gathers 64/128-byte affine bases with 128-bit loads, one ahead of the addition in
//                    flight, folds them into an XYZZ accumulator (8M+2S per point) and closes a run at every
//                    bucket boundary; partial_tree then sums the runs of buckets that have many;
//   4. bucket_merge / bucket_chunk / bucket_bitsums or bucket_tree  sum_b (b+1)*B_b per window: bucket totals, running
//                    sums over chunks of 16 buckets, then a log-depth combination -- no serial 2^(c-1) loop anywhere;
//   5. msm_horner    sum_w 2^(c*w) * S_w in one thread (W*c doublings), leaving one XYZZ partial sum.
//
// Large MSMs over host scalars run steps 1-3 once per chunk of points while the next chunk's scalars upload.
// The affine normalisation / byte encoding (msm_encode) is a separate single-thread kernel so that the
// multi-GPU path can all-gather the 128/256-byte XYZZ partials first (SURVEY.md section 8e).
#include "common.cuh"
#include "tma.cuh"

namespace b200zk {

static constexpr int kMaxWindows = 64;
static constexpr uint32_t kMaxPipelineChunks = 64;  // = events in b200zk_ctx::ev_up
static constexpr int kChunk = 16;  // buckets per running-sum chunk

struct MsmPlan {
  uint32_t c, W, B;       // window bits, windows, buckets per window (2^(c-1))
  uint32_t chunk, T;      // buckets per chunk, chunks per window
  uint32_t merged;        // 1: bases carry precomputed 2^(c*w) multiples, all windows share ONE bucket set
  uint32_t Wr;            // bucket sets to reduce: W, or 1 when merged
  uint32_t table_stride;  // merged: bases of window w start at w * table_stride
};

// window for a precomputed table (all windows share the buckets, so c can be larger: fewer windows)
uint32_t precompute_window(size_t n) {
  uint32_t lg = 0;
  while (((size_t)1 << lg) < n) ++lg;
  // c = 20: a G1 MSM at 2^24 on an H100 SXM (700 W) takes 48.1 / 45.2 / 41.6 / 44.0 ms at c = 18 / 19 / 20 / 21 (beyond
  // 20 the sort over 2^(c-1) buckets and the bucket reduction cost more than the saved window)
  if (lg >= 20) return 20;
  if (lg <= 6) return 6;
  return lg;
}

// scalar_bits: bits the signed-digit recoding must cover = bit length of the group order + 1 (the top window absorbs the
// last carry): 255 for BN254 (r < 2^254), 256 for BLS12-381 (r < 2^255)
static MsmPlan make_plan(size_t n, uint32_t forced_c, uint32_t scalar_bits = 255) {
  uint32_t lg = 0;
  while (((size_t)1 << lg) < n) ++lg;
  // c = 16 for 2^20..2^22 points, 17 from 2^23 up; below that lg-4.  At 2^24 on an H100 SXM at a 400 W power limit a G1
  // MSM over plain bases takes 54.8-54.9 / 52.4-52.8 / 54.9 ms at c = 16 / 17 / 18 (median step, two alternating runs)
  uint32_t c = forced_c ? forced_c : (lg > 8 ? lg - 4 : 4);
  if (!forced_c && c > 16) c = lg >= 23 ? 17 : 16;
  if (c < 2) c = 2;
  if (c > 24) c = 24;
  MsmPlan p;
  p.c = c;
  p.W = (scalar_bits + c - 1) / c;
  p.B = 1u << (c - 1);
  p.chunk = p.B < (uint32_t)kChunk ? p.B : (uint32_t)kChunk;
  p.T = p.B / p.chunk;
  p.merged = 0; p.Wr = p.W; p.table_stride = 0;
  return p;
}

// ---- scalar loading and signed-digit recoding -----------------------------------------------------------
// decode one 32-byte scalar (given as two 128-bit words) into canonical little-endian limbs < r
B2_D void decode_scalar(uint4 lo, uint4 hi, uint32_t flags, uint32_t s[8]) {
  if (flags & B200ZK_SCALARS_BE) {
    s[7] = __byte_perm(lo.x, 0, 0x0123); s[6] = __byte_perm(lo.y, 0, 0x0123); s[5] = __byte_perm(lo.z, 0, 0x0123); s[4] = __byte_perm(lo.w, 0, 0x0123);
    s[3] = __byte_perm(hi.x, 0, 0x0123); s[2] = __byte_perm(hi.y, 0, 0x0123); s[1] = __byte_perm(hi.z, 0, 0x0123); s[0] = __byte_perm(hi.w, 0, 0x0123);
  } else {
    s[0] = lo.x; s[1] = lo.y; s[2] = lo.z; s[3] = lo.w; s[4] = hi.x; s[5] = hi.y; s[6] = hi.z; s[7] = hi.w;
  }
  Fr f;
#pragma unroll
  for (int k = 0; k < 8; ++k) f.v[k] = s[k];
  if (flags & B200ZK_SCALARS_RAW) {
    // another group's scalars (BLS12-381): no reduction; the caller guarantees < r < 2^255 (bls_scalars_check, either byte
    // order).  msm_run_g1 / msm_run_g2 refuse the flag: BN254 scalars are always reduced.
  } else if (flags & B200ZK_SCALARS_MONT) {
    // a Montgomery residue may be any value < 2^256 only if malformed; reduce first so mul's bound holds
#pragma unroll 1
    for (int k = 0; k < 5; ++k) {
      Fr m = Fr::modulus(), t; uint32_t borrow = detail::sub8(t.v, f.v, m.v);
      if (!borrow) f = t;
    }
    f = Fr::from_mont(f);
  } else if (f.v[7] >= FrCfg::mod(7)) {  // top limb below r's: already canonical (every reduced scalar) -- skip the loop
    // 2^256 / r < 6: at most five subtractions bring any 256-bit value below r
#pragma unroll 1
    for (int k = 0; k < 5; ++k) {
      Fr m = Fr::modulus(), t; uint32_t borrow = detail::sub8(t.v, f.v, m.v);
      if (!borrow) f = t;
    }
  }
#pragma unroll
  for (int k = 0; k < 8; ++k) s[k] = f.v[k];
}

// window w of the 256-bit scalar, c <= 24 bits
B2_D uint32_t window_bits(const uint32_t s[8], uint32_t w, uint32_t c) {
  uint32_t bit = w * c;
  uint32_t limb = bit >> 5, off = bit & 31;
  if (limb >= 8) return 0;
  uint64_t v = s[limb];
  if (limb + 1 < 8) v |= (uint64_t)s[limb + 1] << 32;
  return (uint32_t)(v >> off) & ((1u << c) - 1u);
}

// Digit codes: bucket index (0-based) | sign << 31, or kNoDigit for a zero digit.  msm_hist stores them
// window-major (digits[w*n + i]) so that msm_scatter can walk ONE window at a time: all of a window's random
// 4-byte writes then land in that window's slice of idx (n*4 bytes = 64 MiB at 2^24, L2 resident) instead of
// being spread over the whole n*W*4-byte array.
static constexpr uint32_t kNoDigit = 0xffffffffu;

// One atomic per distinct key per warp: hot buckets (top window, scalars 0/1/small) would otherwise serialise
// 32 atomics on one L2 address.  Returns the warp-wide count of `key` and this lane's rank within its group.
// MATCH costs about as many address-divergence-unit cycles as the divergent atomic it saves, so it only runs when the warp shows skew: first count the
// lanes that carry the first active lane's key (one SHFL + one VOTE); fewer than kSkewLanes of them and every lane
// simply is its own group.  Uniform digits (the prover's case) take the cheap path, a hot bucket the exact one.
static constexpr uint32_t kSkewLanes = 3;
B2_D uint32_t warp_group(uint32_t key, bool active, uint32_t* rank, uint32_t* group_mask) {
  const uint32_t full = __activemask();
  const uint32_t act = __ballot_sync(full, active);
  const uint32_t k0 = __shfl_sync(full, key, act ? __ffs(act) - 1 : 0);
  const uint32_t m0 = __ballot_sync(full, active && key == k0);
  if (__popc(m0) < kSkewLanes) {
    *rank = 0;
    *group_mask = 1u << (threadIdx.x & 31);
    return 1;
  }
  uint32_t mask = __match_any_sync(__activemask(), active ? key : kNoDigit);
  uint32_t lane = threadIdx.x & 31;
  *rank = __popc(mask & ((1u << lane) - 1u));
  *group_mask = mask;
  return __popc(mask);
}

// Scalars are streamed through shared memory by the copy engine: each CTA walks tiles of 256 scalars (8 KiB),
// double buffered -- while the warps recode tile k, the bulk copy of tile k+1 is already in flight.
static constexpr uint32_t kHistTile = 256;
__global__ void __launch_bounds__(kHistTile) msm_hist(const void* scalars, size_t n, uint32_t flags, MsmPlan pl, uint32_t* hist, uint32_t* digits) {
  __shared__ __align__(128) uint4 tile[2][kHistTile * 2];
  __shared__ uint64_t bar[2];
  const size_t tiles = (n + kHistTile - 1) / kHistTile;
  if (threadIdx.x == 0) { tma::barrier_init(&bar[0], 1); tma::barrier_init(&bar[1], 1); tma::barrier_init_fence(); }
  __syncthreads();
  auto issue = [&](size_t tl, uint32_t buf) {
    size_t first = tl * kHistTile;
    uint32_t bytes = (uint32_t)((n - first < kHistTile ? n - first : kHistTile) * 32);
    tma::barrier_expect(&bar[buf], bytes);
    tma::bulk_load(tile[buf], reinterpret_cast<const uint8_t*>(scalars) + first * 32, bytes, &bar[buf]);
  };
  if (threadIdx.x == 0 && blockIdx.x < tiles) issue(blockIdx.x, 0);
  uint32_t it = 0;
  for (size_t tl = blockIdx.x; tl < tiles; tl += gridDim.x, ++it) {
    const uint32_t buf = it & 1;
    if (threadIdx.x == 0 && tl + gridDim.x < tiles) issue(tl + gridDim.x, buf ^ 1);  // prefetch the next tile
    tma::barrier_wait(&bar[buf], (it >> 1) & 1);
    const size_t i = tl * kHistTile + threadIdx.x;
    const bool live = i < n;
    uint32_t s[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    if (live) decode_scalar(tile[buf][2 * threadIdx.x], tile[buf][2 * threadIdx.x + 1], flags, s);
    uint32_t carry = 0;
    for (uint32_t w = 0; w < pl.W; ++w) {
      uint32_t coef = window_bits(s, w, pl.c) + carry;
      carry = 0;
      uint32_t neg = 0, mag = coef;
      if (w + 1 < pl.W && coef >= pl.B) { carry = 1; neg = 0x80000000u; mag = (1u << pl.c) - coef; }  // ark make_digits rule
      uint32_t code = mag ? ((mag - 1) | neg) : kNoDigit;
      if (live) digits[(size_t)w * n + i] = code;
      uint32_t rank, gm;
      uint32_t cnt = warp_group(mag - 1, live && mag != 0, &rank, &gm);
      if (live && mag && rank == 0) atomicAdd(&hist[(pl.merged ? 0 : (size_t)w * pl.B) + (mag - 1)], cnt);
    }
    __syncthreads();  // everyone is done with tile[buf] before it is refilled two iterations later
  }
}

// kScatterIlp independent entries per thread per iteration: the slot allocation is an L2 atomic WITH return, i.e. a
// full round trip per entry; with one entry in flight per thread the kernel is latency bound, so each thread keeps
// several allocations in flight.
static constexpr int kScatterIlp = 4;
__global__ void __launch_bounds__(256) msm_scatter(const uint32_t* __restrict__ digits, size_t n, MsmPlan pl, uint32_t* cursor, uint32_t* idx) {
  const size_t total = (size_t)pl.W * n;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  // whole warps stay in the loop together (the bound is padded per warp) so the match/shuffle below is convergent
  const size_t total_pad = (total + 31) & ~(size_t)31;
  for (size_t t0 = blockIdx.x * (size_t)blockDim.x + threadIdx.x; t0 < total_pad; t0 += stride * kScatterIlp) {
    uint32_t code[kScatterIlp], g[kScatterIlp], rank[kScatterIlp], mask[kScatterIlp], base[kScatterIlp];
    size_t w[kScatterIlp];
    bool live[kScatterIlp], active[kScatterIlp];
#pragma unroll
    for (int u = 0; u < kScatterIlp; ++u) {
      const size_t t = t0 + u * stride;
      live[u] = t < total_pad;  // warp-uniform: stride is a multiple of 32
      code[u] = (live[u] && t < total) ? __ldg(digits + t) : kNoDigit;
      active[u] = code[u] != kNoDigit;
      w[u] = live[u] ? t / n : 0;  // a warp may straddle two windows at the seam: key on the global bucket id
      g[u] = (pl.merged ? 0u : (uint32_t)(w[u] * pl.B)) + (code[u] & 0x7fffffffu);
    }
#pragma unroll
    for (int u = 0; u < kScatterIlp; ++u) {
      base[u] = 0; rank[u] = 0; mask[u] = 0;
      if (live[u]) {
        uint32_t cnt = warp_group(g[u], active[u], &rank[u], &mask[u]);
        if (active[u] && rank[u] == 0) base[u] = atomicAdd(&cursor[g[u]], cnt);
      }
    }
#pragma unroll
    for (int u = 0; u < kScatterIlp; ++u) {
      if (live[u]) {
        // broadcast the leader's base to its group: leader = lowest lane of the group
        uint32_t bs = __shfl_sync(mask[u], base[u], __ffs(mask[u]) - 1);
        const size_t t = t0 + u * stride;
        // merged: the entry addresses the precomputed multiple 2^(c*w) * P_i directly
        if (active[u]) idx[bs + rank[u]] = (uint32_t)((t - w[u] * n) + (pl.merged ? w[u] * pl.table_stride : 0)) | (code[u] & 0x80000000u);
      }
    }
  }
}

// ---- two-level sort (r2): tile-local counting sort in shared memory, no per-entry global atomic ------------------------
// The r1 sort paid, per entry, one divergent L2 reduction (msm_hist), one divergent L2 atomic WITH return and one
// divergent 4-byte store (msm_scatter): the SM's address-divergence unit is the limit.
// Here the (window,bucket) key g of an entry is split into a coarse bin (g >> fb) and a fine key (g & (2^fb - 1)):
//   msm_sort_count   every CTA owns a CONTIGUOUS range of scalars; it recodes them (scalar tiles staged by the copy engine,
//                    as in msm_hist) and counts its entries per coarse bin in shared memory -> cnt[bin][cta]
//   (scan)           exclusive scan of cnt in (bin, cta) order: every (bin, cta) pair owns a private, contiguous output run
//   msm_sort_coarse  the same CTA walks the same scalars in tiles of 1024; a tile's entries are ranked per bin with
//                    shared-memory atomics, permuted in shared memory, and copied out so that adjacent lanes write adjacent
//                    addresses (one 8-byte word per entry: value | fine key) -- no global atomics, runs instead of scattered stores
//   msm_sort_fine_*  the bins are cut into segments of 32768 entries (balanced whatever the bin sizes): per-segment fine
//                    histograms in shared memory, a column prefix over each bin's segments (-> the bucket counts, then the
//                    bucket offsets by the ordinary scan), and the final placement staged through shared memory so that a
//                    bucket's entries leave as one run
// Order inside a bucket is not deterministic (shared-memory atomics); the sum is.
static constexpr uint32_t kSortTile = 1024;        // scalars per coarse tile = threads of msm_sort_coarse
static constexpr uint32_t kSortMaxW = 16;          // windows per scalar the staging buffers are sized for (c >= 16)
static constexpr uint32_t kSortMaxBins = 1024;     // coarse bins
static constexpr uint32_t kSortMaxFine = 2048;     // fine keys per bin
static constexpr uint32_t kSortCountSub = 4;
static constexpr int kFineIlp = 8;               // independent (key, value) loads in flight per thread of msm_sort_fine       // msm_sort_count CTAs per coarse CTA range

struct SortPlan {
  uint32_t fb;        // fine bits
  uint32_t C;         // coarse bins = ceil(G / 2^fb)
  uint32_t NC;        // coarse CTAs (ranges of scalars)
  uint32_t range;     // scalars per range (multiple of kSortTile)
  uint32_t G;
};
static bool make_sort_plan(size_t n, const MsmPlan& pl, int sm_count, SortPlan* sp) {
  const size_t G = (size_t)pl.Wr * pl.B;
  uint32_t kb = 0;
  while (((size_t)1 << kb) < G) ++kb;
  if (pl.W > kSortMaxW || kb < 12 || n < ((size_t)1 << 16)) return false;
  uint32_t cb = kb > 19 ? 10 : 9;
  if (kb - cb > 11) return false;  // would need more than kSortMaxFine keys per bin
  sp->fb = kb - cb;
  sp->C = (uint32_t)((G + ((size_t)1 << sp->fb) - 1) >> sp->fb);
  sp->G = (uint32_t)G;
  uint32_t nc = (uint32_t)sm_count;
  size_t tiles = (n + kSortTile - 1) / kSortTile;
  if (nc > tiles) nc = (uint32_t)tiles;
  size_t per = ((tiles + nc - 1) / nc) * kSortTile;
  sp->NC = (uint32_t)((n + per - 1) / per);
  sp->range = (uint32_t)per;
  return true;
}

// digit codes of one scalar: code[w] = bucket | sign << 31, or kNoDigit
// (fully unrolled over kSortMaxW with a guard, so that `code` stays in registers)
B2_D void recode_scalar(const uint32_t s[8], const MsmPlan& pl, uint32_t (&code)[kSortMaxW]) {
  uint32_t carry = 0;
#pragma unroll
  for (uint32_t w = 0; w < kSortMaxW; ++w) {
    code[w] = kNoDigit;
    if (w < pl.W) {
      uint32_t coef = window_bits(s, w, pl.c) + carry;
      carry = 0;
      uint32_t neg = 0, mag = coef;
      if (w + 1 < pl.W && coef >= pl.B) { carry = 1; neg = 0x80000000u; mag = (1u << pl.c) - coef; }  // ark make_digits rule
      code[w] = mag ? ((mag - 1) | neg) : kNoDigit;
    }
  }
}

// grid = NC * kSortCountSub; CTA (r, sub) counts quarter `sub` of range r.  cnt[bin * NC + r] accumulates (zeroed before).
__global__ void __launch_bounds__(kHistTile) msm_sort_count(const void* scalars, size_t n, uint32_t flags, MsmPlan pl, SortPlan sp, uint32_t* cnt) {
  __shared__ __align__(128) uint4 tile[2][kHistTile * 2];
  __shared__ uint64_t bar[2];
  __shared__ uint32_t sh[kSortMaxBins];
  const uint32_t r = blockIdx.x / kSortCountSub, sub = blockIdx.x % kSortCountSub;
  for (uint32_t b = threadIdx.x; b < sp.C; b += kHistTile) sh[b] = 0;
  const size_t lo = (size_t)r * sp.range, hi = lo + sp.range < n ? lo + sp.range : n;
  const size_t tiles_all = lo < hi ? (hi - lo + kHistTile - 1) / kHistTile : 0;
  const size_t per = (tiles_all + kSortCountSub - 1) / kSortCountSub;
  const size_t t0 = sub * per, t1 = t0 + per < tiles_all ? t0 + per : tiles_all;
  if (threadIdx.x == 0) { tma::barrier_init(&bar[0], 1); tma::barrier_init(&bar[1], 1); tma::barrier_init_fence(); }
  __syncthreads();
  auto issue = [&](size_t tl, uint32_t buf) {
    size_t first = lo + tl * kHistTile;
    uint32_t bytes = (uint32_t)((hi - first < kHistTile ? hi - first : kHistTile) * 32);
    tma::barrier_expect(&bar[buf], bytes);
    tma::bulk_load(tile[buf], reinterpret_cast<const uint8_t*>(scalars) + first * 32, bytes, &bar[buf]);
  };
  if (threadIdx.x == 0 && t0 < t1) issue(t0, 0);
  uint32_t it = 0;
  for (size_t tl = t0; tl < t1; ++tl, ++it) {
    const uint32_t buf = it & 1;
    if (threadIdx.x == 0 && tl + 1 < t1) issue(tl + 1, buf ^ 1);
    tma::barrier_wait(&bar[buf], (it >> 1) & 1);
    const size_t i = lo + tl * kHistTile + threadIdx.x;
    if (i < hi) {
      uint32_t s[8], code[kSortMaxW];
      decode_scalar(tile[buf][2 * threadIdx.x], tile[buf][2 * threadIdx.x + 1], flags, s);
      recode_scalar(s, pl, code);
#pragma unroll
      for (uint32_t w = 0; w < kSortMaxW; ++w)
        if (code[w] != kNoDigit) {
          const uint32_t g = (pl.merged ? 0u : w * pl.B) + (code[w] & 0x7fffffffu);
          atomicAdd(&sh[g >> sp.fb], 1u);
        }
    }
    __syncthreads();
  }
  __syncthreads();
  for (uint32_t b = threadIdx.x; b < sp.C; b += kHistTile) if (sh[b]) atomicAdd(&cnt[(size_t)b * sp.NC + r], sh[b]);
}

// grid = NC, block = kSortTile.  base[bin * NC + r] = first output slot of (bin, range r).
struct SortCoarseSmem {
  uint2 ent[kSortTile * kSortMaxW];     // staged entry: x = value (point index | sign << 31), y = fine key
  uint32_t dst[kSortTile * kSortMaxW];  // its slot in the coarse-partitioned array
  uint32_t run_base[kSortMaxBins], tile_cnt[kSortMaxBins], tile_start[kSortMaxBins];
  uint32_t warp_tot[kSortTile / 32];
  uint32_t total;
};
__global__ void __launch_bounds__(kSortTile, 1) msm_sort_coarse(const void* __restrict__ scalars, size_t n, uint32_t flags, MsmPlan pl, SortPlan sp, const uint32_t* __restrict__ base,
                                                               uint2* __restrict__ ent1) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  SortCoarseSmem& sm = *reinterpret_cast<SortCoarseSmem*>(smem_raw);
  const uint32_t r = blockIdx.x, tid = threadIdx.x;
  const size_t lo = (size_t)r * sp.range, hi = lo + sp.range < n ? lo + sp.range : n;
  const uint32_t fmask = (1u << sp.fb) - 1u;
  for (uint32_t b = tid; b < sp.C; b += kSortTile) { sm.run_base[b] = __ldg(base + (size_t)b * sp.NC + r); sm.tile_cnt[b] = 0; }
  __syncthreads();
  const uint4* sc = reinterpret_cast<const uint4*>(scalars);
  for (size_t t0 = lo; t0 < hi; t0 += kSortTile) {
    const size_t i = t0 + tid;
    uint32_t code[kSortMaxW], rank[kSortMaxW];
    const bool live = i < hi;
#pragma unroll
    for (uint32_t w = 0; w < kSortMaxW; ++w) { code[w] = kNoDigit; rank[w] = 0; }
    if (live) {
      uint32_t s[8];
      decode_scalar(__ldg(sc + 2 * i), __ldg(sc + 2 * i + 1), flags, s);
      recode_scalar(s, pl, code);
#pragma unroll
      for (uint32_t w = 0; w < kSortMaxW; ++w)
        if (code[w] != kNoDigit) {
          const uint32_t g = (pl.merged ? 0u : w * pl.B) + (code[w] & 0x7fffffffu);
          rank[w] = atomicAdd(&sm.tile_cnt[g >> sp.fb], 1u);
        }
    }
    __syncthreads();
    // exclusive scan of tile_cnt over the C <= 1024 bins: one bin per thread
    {
      const uint32_t v = tid < sp.C ? sm.tile_cnt[tid] : 0;
      uint32_t incl = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if ((tid & 31) >= (unsigned)o) incl += t; }
      if ((tid & 31) == 31) sm.warp_tot[tid >> 5] = incl;
      __syncthreads();
      uint32_t wb = 0;
      for (uint32_t k = 0; k < (tid >> 5); ++k) wb += sm.warp_tot[k];
      if (tid < sp.C) sm.tile_start[tid] = wb + incl - v;
      if (tid == kSortTile - 1) sm.total = wb + incl;
    }
    __syncthreads();
    if (live) {
#pragma unroll
      for (uint32_t w = 0; w < kSortMaxW; ++w)
        if (code[w] != kNoDigit) {
          const uint32_t g = (pl.merged ? 0u : w * pl.B) + (code[w] & 0x7fffffffu);
          const uint32_t b = g >> sp.fb, pos = sm.tile_start[b] + rank[w];
          // merged: the entry addresses the precomputed multiple 2^(c*w) * P_i directly
          sm.ent[pos] = make_uint2((uint32_t)(i + (pl.merged ? (size_t)w * pl.table_stride : 0)) | (code[w] & 0x80000000u), g & fmask);
          sm.dst[pos] = sm.run_base[b] + rank[w];
        }
    }
    __syncthreads();
    const uint32_t total = sm.total;
    for (uint32_t t = tid; t < total; t += kSortTile) ent1[sm.dst[t]] = sm.ent[t];  // adjacent t: same bin's run, adjacent slots
    __syncthreads();
    if (tid < sp.C) { sm.run_base[tid] += sm.tile_cnt[tid]; sm.tile_cnt[tid] = 0; }
    __syncthreads();
  }
}

// ---- fine pass, balanced: work items are SEGMENTS of kFineSeg entries of a coarse bin ------------------------------------
// One CTA per coarse bin would be as unbalanced as the bins are -- and they are: the top window of a 254-bit scalar
// only has 254 - 240 = 14 bits at c = 20, so all of its 2^24 entries land in the 16 lowest bins (3.5x the average; at
// c = 19 / 21 / 22 in one or two bins), and skewed witnesses do the same to any bin.  Now:
//   msm_sort_items     item_start[b] = sum_{b' < b} ceil(size(b') / kFineSeg)                          (one small CTA)
//   msm_sort_fine_count  item i = (bin, segment): histogram of its entries' fine keys -> cnt2[i][key]
//   msm_sort_fine_prefix thread (bin, key): exclusive prefix of cnt2[.][key] over the bin's segments, total -> hist[g]
//   (scan of hist -> offsets, the kernels the legacy sort used)
//   msm_sort_fine_place  item i: cursor[key] = offsets[g] + cnt2[i][key]; staged placement of its segment
static constexpr uint32_t kFineTile = 8192;   // entries per staged tile = 8 per thread
static constexpr uint32_t kFineSeg = 4 * kFineTile;  // entries per work item
struct SortFineSmem {
  uint32_t val[kFineTile], dst[kFineTile];
  uint32_t cur[kSortMaxFine], tcnt[kSortMaxFine], tstart[kSortMaxFine];
  uint32_t warp_tot[32];
  uint32_t total;
};
// exclusive scan of in[0..F) (F <= 2048, two keys per thread of a 1024-thread CTA) into out; leaves the grand total in *total
B2_D void scan_fine_keys(const uint32_t* in, uint32_t* out, uint32_t F, uint32_t* warp_tot, uint32_t* total) {
  const uint32_t tid = threadIdx.x, k0 = 2 * tid, k1 = 2 * tid + 1;
  const uint32_t v0 = k0 < F ? in[k0] : 0, v1 = k1 < F ? in[k1] : 0;
  uint32_t incl = v0 + v1;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if ((tid & 31) >= (unsigned)o) incl += t; }
  if ((tid & 31) == 31) warp_tot[tid >> 5] = incl;
  __syncthreads();
  uint32_t wb = 0;
  for (uint32_t k = 0; k < (tid >> 5); ++k) wb += warp_tot[k];
  const uint32_t ex = wb + incl - v0 - v1;
  if (k0 < F) out[k0] = ex;
  if (k1 < F) out[k1] = ex + v0;
  if (tid == 1023) *total = wb + incl;
  __syncthreads();
}
// one CTA of 1024 threads: item_start[0..C] (C <= 1024)
__global__ void __launch_bounds__(1024) msm_sort_items(const uint32_t* __restrict__ base, SortPlan sp, uint32_t* __restrict__ item_start) {
  __shared__ uint32_t wt[32];
  const uint32_t tid = threadIdx.x;
  uint32_t v = 0;
  if (tid < sp.C) { const uint32_t sz = __ldg(base + (size_t)(tid + 1) * sp.NC) - __ldg(base + (size_t)tid * sp.NC); v = (sz + kFineSeg - 1) / kFineSeg; }
  uint32_t incl = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if ((tid & 31) >= (unsigned)o) incl += t; }
  if ((tid & 31) == 31) wt[tid >> 5] = incl;
  __syncthreads();
  uint32_t wb = 0;
  for (uint32_t k = 0; k < (tid >> 5); ++k) wb += wt[k];
  if (tid < sp.C) item_start[tid] = wb + incl - v;
  if (tid == sp.C - 1) item_start[sp.C] = wb + incl;
}
// the bin of item i: largest b with item_start[b] <= i (items of empty bins do not exist: item_start repeats)
B2_D uint32_t item_bin(const uint32_t* __restrict__ item_start, uint32_t C, uint32_t i) {
  uint32_t lo = 0, hi = C;
  while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (__ldg(item_start + mid) <= i) lo = mid; else hi = mid; }
  return lo;
}
__global__ void __launch_bounds__(1024, 2) msm_sort_fine_count(const uint2* __restrict__ ent1, SortPlan sp, const uint32_t* __restrict__ base, const uint32_t* __restrict__ item_start,
                                                               uint32_t* __restrict__ cnt2) {
  __shared__ uint32_t fh[kSortMaxFine];
  const uint32_t i = blockIdx.x, tid = threadIdx.x, F = 1u << sp.fb;
  if (i >= __ldg(item_start + sp.C)) return;
  const uint32_t b = item_bin(item_start, sp.C, i);
  const uint32_t bs = __ldg(base + (size_t)b * sp.NC), be = __ldg(base + (size_t)(b + 1) * sp.NC);
  const uint32_t s0 = bs + (i - __ldg(item_start + b)) * kFineSeg, s1 = (be - s0 > kFineSeg) ? s0 + kFineSeg : be;
  for (uint32_t k = tid; k < F; k += 1024) fh[k] = 0;
  __syncthreads();
  for (uint32_t e0 = s0 + tid; e0 < s1; e0 += 1024 * kFineIlp) {
    uint32_t kk[kFineIlp];
#pragma unroll
    for (int u = 0; u < kFineIlp; ++u) { const uint32_t e = e0 + u * 1024; kk[u] = e < s1 ? __ldg(&ent1[e].y) : 0xffffffffu; }
#pragma unroll
    for (int u = 0; u < kFineIlp; ++u) if (kk[u] != 0xffffffffu) atomicAdd(&fh[kk[u]], 1u);
  }
  __syncthreads();
  for (uint32_t k = tid; k < F; k += 1024) cnt2[(size_t)i * F + k] = fh[k];
}
// grid = C * F / 256 threads: thread (b, key) turns cnt2[item][key] into its exclusive prefix over the bin's items
__global__ void __launch_bounds__(256) msm_sort_fine_prefix(SortPlan sp, const uint32_t* __restrict__ item_start, uint32_t* __restrict__ cnt2, uint32_t* __restrict__ hist) {
  const uint32_t F = 1u << sp.fb;
  const size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (t >= (size_t)sp.C * F) return;
  const uint32_t b = (uint32_t)(t >> sp.fb), k = (uint32_t)t & (F - 1);
  const uint32_t i0 = __ldg(item_start + b), i1 = __ldg(item_start + b + 1);
  uint32_t run = 0;
  for (uint32_t i = i0; i < i1; ++i) {
    const size_t at = (size_t)i * F + k;
    const uint32_t c = cnt2[at];
    cnt2[at] = run;
    run += c;
  }
  if (t < sp.G) hist[t] = run;
}
__global__ void __launch_bounds__(1024, 1) msm_sort_fine_place(const uint2* __restrict__ ent1, SortPlan sp, const uint32_t* __restrict__ base, const uint32_t* __restrict__ item_start,
                                                               const uint32_t* __restrict__ cnt2, const uint32_t* __restrict__ offsets, uint32_t* __restrict__ idx) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  SortFineSmem& sm = *reinterpret_cast<SortFineSmem*>(smem_raw);
  const uint32_t i = blockIdx.x, tid = threadIdx.x, F = 1u << sp.fb;
  if (i >= __ldg(item_start + sp.C)) return;
  const uint32_t b = item_bin(item_start, sp.C, i);
  const uint32_t bs = __ldg(base + (size_t)b * sp.NC), be = __ldg(base + (size_t)(b + 1) * sp.NC);
  const uint32_t s0 = bs + (i - __ldg(item_start + b)) * kFineSeg, s1 = (be - s0 > kFineSeg) ? s0 + kFineSeg : be;
  for (uint32_t k = tid; k < F; k += 1024) {
    const size_t g = (size_t)b * F + k;
    sm.cur[k] = (g < sp.G ? __ldg(offsets + g) : 0u) + __ldg(cnt2 + (size_t)i * F + k);  // absolute slot of this item's first entry of key k
    sm.tcnt[k] = 0;
  }
  __syncthreads();
  for (uint32_t t0 = s0; t0 < s1; t0 += kFineTile) {
    uint2 ev[kFineTile / 1024];
    uint32_t rank[kFineTile / 1024];
#pragma unroll
    for (int u = 0; u < (int)(kFineTile / 1024); ++u) {
      const uint32_t e = t0 + u * 1024 + tid;
      ev[u] = e < s1 ? __ldg(ent1 + e) : make_uint2(0u, 0xffffffffu);
    }
#pragma unroll
    for (int u = 0; u < (int)(kFineTile / 1024); ++u) rank[u] = ev[u].y != 0xffffffffu ? atomicAdd(&sm.tcnt[ev[u].y], 1u) : 0u;
    __syncthreads();
    scan_fine_keys(sm.tcnt, sm.tstart, F, sm.warp_tot, &sm.total);
#pragma unroll
    for (int u = 0; u < (int)(kFineTile / 1024); ++u)
      if (ev[u].y != 0xffffffffu) {
        const uint32_t pos = sm.tstart[ev[u].y] + rank[u];
        sm.val[pos] = ev[u].x;
        sm.dst[pos] = sm.cur[ev[u].y] + rank[u];
      }
    __syncthreads();
    const uint32_t total = sm.total;
    for (uint32_t t = tid; t < total; t += 1024) idx[sm.dst[t]] = sm.val[t];  // adjacent t: one bucket's run, adjacent slots
    __syncthreads();
    for (uint32_t k = tid; k < F; k += 1024) { sm.cur[k] += sm.tcnt[k]; sm.tcnt[k] = 0; }
    __syncthreads();
  }
}

// ---- exclusive scan of the histogram (G entries) ---------------------------------------------------------
static constexpr int kScanThreads = 256, kScanItems = 8, kScanTile = kScanThreads * kScanItems;

// seg == 0: scan the counts themselves (-> bucket offsets).
// seg  > 0: scan the flag "bucket i is non-empty and does not start on a multiple of seg" (aux = bucket offsets);
//           scan_apply then adds ceil(offset/seg), giving run_off[i] = index of the first RUN of bucket i when the
//           sorted entries are cut at every multiple of seg and at every bucket start (see msm_accumulate).
B2_D uint32_t scan_value(const uint32_t* in, const uint32_t* aux, size_t i, uint32_t seg) {
  uint32_t v = in[i];
  if (!seg) return v;
  return (v != 0 && (aux[i] % seg) != 0) ? 1u : 0u;
}

__global__ void __launch_bounds__(kScanThreads) scan_tile_sums(const uint32_t* in, const uint32_t* aux, size_t G, uint32_t seg, uint32_t* tile_sums) {
  __shared__ uint32_t red[kScanThreads / 32];
  size_t base = (size_t)blockIdx.x * kScanTile + (size_t)threadIdx.x * kScanItems;
  uint32_t s = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) if (base + k < G) s += scan_value(in, aux, base + k, seg);
#pragma unroll
  for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = s;
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t t = 0;
    for (int k = 0; k < kScanThreads / 32; ++k) t += red[k];
    tile_sums[blockIdx.x] = t;
  }
}
__global__ void __launch_bounds__(1024) scan_tile_offsets(uint32_t* tile_sums, size_t tiles) {
  // single block: exclusive scan of up to a few thousand tile sums, 1024 at a time
  __shared__ uint32_t buf[1024];
  __shared__ uint32_t carry;
  if (threadIdx.x == 0) carry = 0;
  __syncthreads();
  for (size_t base = 0; base < tiles; base += 1024) {
    size_t i = base + threadIdx.x;
    uint32_t v = i < tiles ? tile_sums[i] : 0;
    buf[threadIdx.x] = v;
    __syncthreads();
    for (int o = 1; o < 1024; o <<= 1) {
      uint32_t t = threadIdx.x >= (unsigned)o ? buf[threadIdx.x - o] : 0;
      __syncthreads();
      buf[threadIdx.x] += t;
      __syncthreads();
    }
    uint32_t incl = buf[threadIdx.x], c0 = carry;
    __syncthreads();
    if (i < tiles) tile_sums[i] = c0 + incl - v;
    if (threadIdx.x == 1023) carry = c0 + incl;
    __syncthreads();
  }
}
__global__ void __launch_bounds__(kScanThreads) scan_apply(const uint32_t* in, const uint32_t* aux, size_t G, uint32_t seg, const uint32_t* tile_offsets, uint32_t* offsets, uint32_t* cursor) {
  __shared__ uint32_t warp_tot[kScanThreads / 32];
  size_t base = (size_t)blockIdx.x * kScanTile + (size_t)threadIdx.x * kScanItems;
  uint32_t v[kScanItems], s = 0;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) { v[k] = base + k < G ? scan_value(in, aux, base + k, seg) : 0; s += v[k]; }
  uint32_t incl = s;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, incl, o); if ((threadIdx.x & 31) >= (unsigned)o) incl += t; }
  if ((threadIdx.x & 31) == 31) warp_tot[threadIdx.x >> 5] = incl;
  __syncthreads();
  uint32_t wbase = 0;
  for (unsigned k = 0; k < (threadIdx.x >> 5); ++k) wbase += warp_tot[k];
  uint32_t run = tile_offsets[blockIdx.x] + wbase + incl - s;
#pragma unroll
  for (int k = 0; k < kScanItems; ++k) {
    if (base + k < G) { offsets[base + k] = seg ? run + (aux[base + k] + seg - 1) / seg : run; if (cursor) cursor[base + k] = run; }
    run += v[k];
  }
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == kScanThreads - 1) offsets[G] = seg ? run + (aux[G] + seg - 1) / seg : run;  // total
}

// ---- bucket accumulation ----------------------------------------------------------------------------------
// Buckets are wildly uneven even for uniform scalars (the top window of a 254-bit scalar only has
// 254 - (W-1)c bits, and real witnesses are full of 0/1 values), so work is NOT split by bucket.  The sorted
// entry array is cut into fixed slices of kSegLen entries, one per thread: every thread performs exactly
// kSegLen gathers + mixed additions, whatever the bucket sizes.  Inside its slice a thread closes a RUN (stores
// the XYZZ partial and its bucket id) whenever the bucket changes.  Runs are numbered along the sorted order:
// a run starts at every multiple of kSegLen and at every bucket start, so the first run of bucket g is
//   run_off[g] = ceil(offsets[g]/kSegLen) + #{non-empty g' < g : offsets[g'] % kSegLen != 0}     (scan, seg mode)
// and a thread derives its first slot from the same formula.  partial_tree then folds the runs of every bucket
// that has more than one (a bucket straddling a slice boundary, or a heavy bucket spanning many slices) with a
// radix-kTreeRadix tree in place, leaving each bucket's total in its first run.
static constexpr uint32_t kSegLenMax = 256;  // the slice length itself is a launch parameter (wave balancing)
static constexpr uint32_t kTreeRadix = 64;
// Buckets with at most kDirectRuns runs are NOT folded by partial_tree: their consumers (bucket_chunk, bucket_merge) add
// the runs themselves.  With slices of ~240 entries and buckets of ~416 (c = 20 at 2^24) nearly every bucket has 2-3 runs:
// folding them in the tree kernel keeps only one lane in 2-3 busy; the consumers walk buckets anyway.  The tree only remains for heavy buckets (skewed scalars).
static constexpr uint32_t kDirectRuns = 4;

// Slice length for M entries: every thread does the same work, so the launch runs in lock-step "waves" of
// `resident` threads; pick the length that fills a whole number of waves instead of leaving the last one part empty.
static uint32_t pick_slice_len(size_t M, size_t resident) {
  if (M == 0) return kSegLenMax;
  size_t per_thread = (M + resident - 1) / resident;            // entries per thread if it were a single wave
  size_t waves = (per_thread + kSegLenMax - 1) / kSegLenMax;
  size_t len = (M + resident * waves - 1) / (resident * waves);
  if (len < 16) len = 16;
  if (len > kSegLenMax) len = kSegLenMax;
  return (uint32_t)len;
}

// largest g in [lo, G) with offsets[g] <= e, given offsets[lo] <= e: gallop then bisect (the next non-empty
// bucket is almost always within a few entries; empty buckets repeat the same offset and are skipped)
B2_D uint32_t bucket_of(const uint32_t* __restrict__ offsets, uint32_t G, uint32_t lo, uint32_t e) {
  uint32_t step = 1, hi = lo + 1;
  while (hi < G && __ldg(offsets + hi) <= e) { lo = hi; step <<= 1; hi = lo + step; }
  if (hi > G) hi = G;
  // invariant: offsets[lo] <= e, and (hi == G or offsets[hi] > e)
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (__ldg(offsets + mid) <= e) lo = mid; else hi = mid;
  }
  return lo;
}

// sorted entry e is idx[e] = base index | sign << 31 into the bases / window table
template <class F>
__global__ void __launch_bounds__(128, 1) msm_accumulate(const void* __restrict__ points, const uint32_t* __restrict__ idx,
                                                      const uint32_t* __restrict__ offsets, const uint32_t* __restrict__ run_off,
                                                      uint32_t G, uint32_t kSegLen, void* __restrict__ partials, uint32_t* __restrict__ run_bucket) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t M = __ldg(offsets + G);
  const uint64_t e0_64 = (uint64_t)t * kSegLen;
  if (e0_64 >= M) return;
  const uint32_t e0 = (uint32_t)e0_64;
  const uint32_t e1 = (M - e0 > kSegLen) ? e0 + kSegLen : M;
  // full binary search once per thread
  uint32_t g;
  {
    uint32_t lo = 0, hi = G;
    while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (__ldg(offsets + mid) <= e0) lo = mid; else hi = mid; }
    g = lo;
  }
  const uint32_t off0 = __ldg(offsets + g);
  uint32_t slot = t + (__ldg(run_off + g) - (off0 + kSegLen - 1) / kSegLen) + ((off0 % kSegLen) ? 1u : 0u);
  uint32_t next = __ldg(offsets + g + 1);  // first entry of the following bucket (> e0)
  XYZZ<F> acc = XYZZ<F>::identity();
  uint32_t v = __ldg(idx + e0);
  Affine<F> p = load_affine_nc<F>(points, v & 0x7fffffffu);
  for (uint32_t e = e0; e < e1; ++e) {
    // software prefetch: issue the next gather before the ~1500-instruction addition
    uint32_t vn = v; Affine<F> pn = p;
    if (e + 1 < e1) { vn = __ldg(idx + e + 1); pn = load_affine_nc<F>(points, vn & 0x7fffffffu); }
    if (e == next) {  // bucket boundary: close the run
      store_xyzz(partials, slot, acc);
      run_bucket[slot] = g;
      ++slot;
      acc = XYZZ<F>::identity();
      g = bucket_of(offsets, G, g + 1, e);
      next = __ldg(offsets + g + 1);
    }
    if (v >> 31) p.y = F::neg(p.y);
    xyzz_add_mixed(acc, p.x, p.y);
    v = vn; p = pn;
  }
  store_xyzz(partials, slot, acc);
  run_bucket[slot] = g;
}

// ---- G2 accumulation on lane pairs -----------------------------------------------------------------------------
// msm_accumulate<Fq2> keeps an XYZZ accumulator over Fq2 (64 registers), the point and its prefetch (2 x 32) and the
// temporaries of an Fq2 product in ONE thread: 255 registers, 2 CTAs (8 warps) per SM, too few warps to cover the
// carry chains' latency.  Here two adjacent lanes share one slice: lane 2k holds the real component (c0) of every Fq2 value,
// lane 2k+1 the imaginary one (c1) -- half the registers per thread, the occupancy of the G1 kernel -- and the
// components an Fq2 product needs from the partner lane travel by SHFL.XOR 1 (8 shuffles per value, ~90 per mixed
// addition against ~1800 wide multiplies per lane).  Every product stays a shared-reduction form of field.cuh:
//   (a b).c0 = a0 b0 + (-a1) b1      (a b).c1 = a1 b0 + a0 b1            one mul2_add per lane
//   (a^2).c0 = (a0 + a1)(a0 - a1)    (a^2).c1 = (2 a1) a0                one mul per lane
//   (a b - c d).c0 / .c1                                                  one mul4_add per lane
// Operands are chosen with selects on the lane's role, so both lanes run the same instruction stream; pair-uniform
// branches (identity, doubling, cancellation) are decided on both components with one more shuffle.  Memory layout,
// slice scheme and run numbering are those of msm_accumulate: the other kernels do not know the difference.
// The three products of the lane-pair kernel as REAL functions (arguments and result travel in registers: checked in SASS,
// no local-memory traffic).  Inlined, one G2 mixed addition is ~3500 SASS instructions = 56 KB and the loop body does not
// fit the instruction cache (instruction-cache misses were the top stall); as calls the body is ~13 KB plus
// ~13 KB of callees, the size of the G1 kernel's body.
// One product per call: callees that compute the two independent products the formulas offer at every step (U2 | S2,
// PP | R^2, PPP | Q, ZZ3 | ZZZ3) lose: marshalling 64 argument registers per call costs more than the second carry
// chain per warp gains.
__device__ __noinline__ Fq fq_mul_call(Fq a, Fq b) { return Fq::mul(a, b); }
__device__ __noinline__ Fq fq_mul2_add_call(Fq a, Fq b, Fq c, Fq d) { return Fq::mul2_add(a, b, c, d); }
__device__ __noinline__ Fq fq_mul4_add_call(Fq a, Fq b, Fq c, Fq d, Fq e, Fq f, Fq g, Fq h) { return Fq::mul4_add(a, b, c, d, e, f, g, h); }

struct PairLane {
  uint32_t mask;  // the two lanes of this pair
  bool hi;        // this lane holds c1
  B2_D Fq partner(const Fq& a) const {
    Fq r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.v[i] = __shfl_xor_sync(mask, a.v[i], 1);
    return r;
  }
  B2_D bool both(bool mine) const { return __shfl_xor_sync(mask, mine ? 1u : 0u, 1) != 0 && mine; }
  B2_D Fq sel(const Fq& if_hi, const Fq& if_lo) const {
    Fq r;
#pragma unroll
    for (int i = 0; i < 8; ++i) r.v[i] = hi ? if_hi.v[i] : if_lo.v[i];
    return r;
  }
  // component of a * b; pa / pb = the partner's component of a / b
  B2_D Fq mul(const Fq& a, const Fq& pa, const Fq& b, const Fq& pb) const {
    // lo: a b + (-pa) pb      hi: a pb + pa b
    return fq_mul2_add_call(a, sel(pb, b), sel(pa, Fq::neg(pa)), sel(b, pb));
  }
  B2_D Fq sqr(const Fq& a, const Fq& pa) const {
    // lo: (a + pa)(a - pa)    hi: (2 a) pa
    return fq_mul_call(sel(Fq::dbl(a), Fq::add(a, pa)), sel(pa, Fq::sub(a, pa)));
  }
  // component of a * b - c * d
  B2_D Fq mul2_sub(const Fq& a, const Fq& pa, const Fq& b, const Fq& pb, const Fq& c, const Fq& pc, const Fq& d, const Fq& pd) const {
    // lo: a b + (-pa) pb + (-c) d + pc pd      hi: pa b + a pb + (-pc) d + (-c) pd
    const Fq nc = Fq::neg(c);
    return fq_mul4_add_call(sel(pa, a), b, sel(a, Fq::neg(pa)), pb, sel(Fq::neg(pc), nc), d, sel(nc, pc), pd);
  }
  B2_D Fq one() const { return hi ? Fq::zero() : Fq::one(); }
};
struct XYZZHalf { Fq x, y, zz, zzz; };  // one component of an XYZZ<Fq2>

// acc = 2 * (x1, y1), affine input (mdbl-2008-s-1, a = 0)
B2_D void pair_mdbl(const PairLane& L, XYZZHalf& acc, const Fq& x1, const Fq& y1) {
  const Fq U = Fq::dbl(y1), pU = L.partner(U);
  const Fq V = L.sqr(U, pU), pV = L.partner(V);
  const Fq W = L.mul(U, pU, V, pV), pW = L.partner(W);
  const Fq px1 = L.partner(x1), py1 = L.partner(y1);
  const Fq S = L.mul(x1, px1, V, pV);
  const Fq xx = L.sqr(x1, px1), M = Fq::add(Fq::dbl(xx), xx), pM = L.partner(M);
  acc.x = Fq::sub(L.sqr(M, pM), Fq::dbl(S));
  const Fq T = Fq::sub(S, acc.x), pT = L.partner(T);
  acc.y = L.mul2_sub(M, pM, T, pT, W, pW, y1, py1);
  acc.zz = V; acc.zzz = W;
}
// acc += (x2, y2)   (madd-2008-s; identity, doubling and cancellation handled; decisions are pair-uniform)
B2_D void pair_add_mixed(const PairLane& L, XYZZHalf& acc, const Fq& x2, const Fq& y2) {
  if (L.both(x2.is_zero() && y2.is_zero())) return;
  if (L.both(acc.zz.is_zero())) { acc.x = x2; acc.y = y2; acc.zz = L.one(); acc.zzz = L.one(); return; }
  const Fq pzz = L.partner(acc.zz), pzzz = L.partner(acc.zzz);
  const Fq U2 = L.mul(x2, L.partner(x2), acc.zz, pzz), S2 = L.mul(y2, L.partner(y2), acc.zzz, pzzz);
  const Fq P = Fq::sub(U2, acc.x), R = Fq::sub(S2, acc.y);
  if (L.both(P.is_zero())) {
    if (L.both(R.is_zero())) pair_mdbl(L, acc, x2, y2);
    else { acc.x = Fq::zero(); acc.y = Fq::zero(); acc.zz = Fq::zero(); acc.zzz = Fq::zero(); }
    return;
  }
  const Fq pP = L.partner(P);
  const Fq PP = L.sqr(P, pP), pPP = L.partner(PP);
  const Fq PPP = L.mul(P, pP, PP, pPP), pPPP = L.partner(PPP);
  const Fq Q = L.mul(acc.x, L.partner(acc.x), PP, pPP);
  const Fq pR = L.partner(R);
  const Fq x3 = Fq::sub(Fq::sub(L.sqr(R, pR), PPP), Fq::dbl(Q));
  const Fq T = Fq::sub(Q, x3), pT = L.partner(T);
  acc.y = L.mul2_sub(R, pR, T, pT, acc.y, L.partner(acc.y), PPP, pPPP);
  acc.x = x3;
  acc.zz = L.mul(acc.zz, pzz, PP, pPP);
  acc.zzz = L.mul(acc.zzz, pzzz, PPP, pPPP);
}

// One thread PAIR per slice of kSegLen sorted entries; blockDim.x threads = blockDim.x / 2 slices.  Compiled for
// kG2PairBlocks CTAs per SM: 154 registers, no spills.  At 4 CTAs per SM (128 registers, spills) a G2 MSM at 2^24 on an
// H100 SXM at a 400 W power limit took 138.6-143.8 ms against 134.8 ms at 3 (median step, two alternating runs each).
static constexpr unsigned kG2PairBlocks = 3;
__global__ void __launch_bounds__(128, kG2PairBlocks) msm_accumulate_g2_pair(const void* __restrict__ points, const uint32_t* __restrict__ idx, const uint32_t* __restrict__ offsets,
                                                                const uint32_t* __restrict__ run_off, uint32_t G, uint32_t kSegLen, void* __restrict__ partials,
                                                                uint32_t* __restrict__ run_bucket) {
  const uint32_t gt = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t t = gt >> 1;
  PairLane L;
  L.hi = (threadIdx.x & 1) != 0;
  L.mask = 3u << (threadIdx.x & 30);
  const uint32_t M = __ldg(offsets + G);
  const uint64_t e0_64 = (uint64_t)t * kSegLen;
  if (e0_64 >= M) return;  // pair-uniform
  const uint32_t e0 = (uint32_t)e0_64;
  const uint32_t e1 = (M - e0 > kSegLen) ? e0 + kSegLen : M;
  uint32_t g;
  {
    uint32_t lo = 0, hi = G;
    while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (__ldg(offsets + mid) <= e0) lo = mid; else hi = mid; }
    g = lo;
  }
  const uint32_t off0 = __ldg(offsets + g);
  uint32_t slot = t + (__ldg(run_off + g) - (off0 + kSegLen - 1) / kSegLen) + ((off0 % kSegLen) ? 1u : 0u);
  uint32_t next = __ldg(offsets + g + 1);
  // affine G2 point = x.c0 | x.c1 | y.c0 | y.c1 (4 x 32 B): this lane's components sit at words 0 + hi and 2 + hi
  const uint32_t comp = L.hi ? 1u : 0u;
  auto load_half = [&](uint32_t v, Fq& x, Fq& y) {
    const size_t w = 4 * (size_t)(v & 0x7fffffffu) + comp;
    x = load_fe_nc<Fq>(points, w);
    y = load_fe_nc<Fq>(points, w + 2);
  };
  // XYZZ<Fq2> partial = 8 words: x.c0 x.c1 y.c0 y.c1 zz.c0 zz.c1 zzz.c0 zzz.c1
  auto store_half = [&](uint32_t s, const XYZZHalf& a) {
    const size_t w = 8 * (size_t)s + comp;
    store_fe<Fq>(partials, w, a.x); store_fe<Fq>(partials, w + 2, a.y); store_fe<Fq>(partials, w + 4, a.zz); store_fe<Fq>(partials, w + 6, a.zzz);
  };
  XYZZHalf acc = {Fq::zero(), Fq::zero(), Fq::zero(), Fq::zero()};
  // The next point is prefetched into L2 (prefetch.global.L2), not into registers: with the 16 registers of a register
  // prefetch the kernel needs 168+ registers; an addition (~1800 wide multiplies per lane) is long enough for the other
  // warps to cover an L2 hit.
  auto prefetch_half = [&](uint32_t v) {
    const uint8_t* q = reinterpret_cast<const uint8_t*>(points) + (4 * (size_t)(v & 0x7fffffffu) + comp) * 32;
    asm volatile("prefetch.global.L2 [%0];" ::"l"(q));
    asm volatile("prefetch.global.L2 [%0];" ::"l"(q + 64));
  };
  uint32_t v = __ldg(idx + e0);
  prefetch_half(v);
  for (uint32_t e = e0; e < e1; ++e) {
    uint32_t vn = v;
    if (e + 1 < e1) { vn = __ldg(idx + e + 1); prefetch_half(vn); }
    if (e == next) {  // bucket boundary: close the run
      store_half(slot, acc);
      if (!L.hi) run_bucket[slot] = g;
      ++slot;
      acc = {Fq::zero(), Fq::zero(), Fq::zero(), Fq::zero()};
      g = bucket_of(offsets, G, g + 1, e);
      next = __ldg(offsets + g + 1);
    }
    Fq px, py;
    load_half(v, px, py);
    if (v >> 31) py = Fq::neg(py);  // -(y0 + y1 u) = -y0 + (-y1) u: component-wise
    pair_add_mixed(L, acc, px, py);
    v = vn;
  }
  store_half(slot, acc);
  if (!L.hi) run_bucket[slot] = g;
}

template <class F>
__global__ void __launch_bounds__(128) partial_tree(const uint32_t* __restrict__ seg_off, const uint32_t* __restrict__ seg_bucket, uint32_t G,
                                                    uint32_t stride, void* __restrict__ partials) {
  uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= __ldg(seg_off + G)) return;
  const uint32_t g = seg_bucket[s];
  const uint32_t base = __ldg(seg_off + g), ns = __ldg(seg_off + g + 1) - base, j = s - base;
  if (ns <= kDirectRuns || ns <= stride || (j % (stride * kTreeRadix)) != 0) return;
  XYZZ<F> acc = load_xyzz<F>(partials, s);
  for (uint32_t t = 1; t < kTreeRadix; ++t) {
    uint32_t jj = j + t * stride;
    if (jj >= ns) break;
    XYZZ<F> q = load_xyzz<F>(partials, s + t * stride);
    xyzz_add(acc, q);
  }
  store_xyzz(partials, s, acc);
}

// total of a non-empty bucket whose runs start at `so`: its first run (already folded by partial_tree when it had more than
// kDirectRuns runs), else the sum of its `cnt` runs
template <class F> B2_D XYZZ<F> bucket_total(const void* __restrict__ partials, uint32_t so, uint32_t cnt) {
  XYZZ<F> b = load_xyzz<F>(partials, so);
  if (cnt <= kDirectRuns)
    for (uint32_t r = 1; r < cnt; ++r) { XYZZ<F> q = load_xyzz<F>(partials, so + r); xyzz_add(b, q); }
  return b;
}

// totals[g] (+)= this chunk's total of bucket g (its first run after partial_tree); first chunk initialises
template <class F>
__global__ void __launch_bounds__(128) bucket_merge(const void* __restrict__ partials, const uint32_t* __restrict__ run_off, uint32_t G, int first, void* __restrict__ totals) {
  uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  uint32_t so = __ldg(run_off + g);
  const uint32_t cnt = __ldg(run_off + g + 1) - so;
  bool has = cnt != 0;
  if (first) {
    store_xyzz(totals, g, has ? bucket_total<F>(partials, so, cnt) : XYZZ<F>::identity());
  } else if (has) {
    XYZZ<F> t = load_xyzz<F>(totals, g), p = bucket_total<F>(partials, so, cnt);
    xyzz_add(t, p);
    store_xyzz(totals, g, t);
  }
}

// ---- bucket reduction: S_w = sum_b (b+1) * B[w][b] ---------------------------------------------------------
// chunk j of window w: S = sum B, V = sum_k (k+1) * B[j*chunk + k]
template <class F>
__global__ void __launch_bounds__(128) bucket_chunk(const void* __restrict__ partials, const uint32_t* __restrict__ seg_off, MsmPlan pl, void* __restrict__ chunkS, void* __restrict__ chunkV) {
  size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  size_t total = (size_t)pl.Wr * pl.T;
  if (t >= total) return;
  size_t first = t * pl.chunk;  // bucket arrays are [w][b] contiguous and T*chunk == B
  XYZZ<F> run = XYZZ<F>::identity(), acc = XYZZ<F>::identity();
  for (int k = (int)pl.chunk - 1; k >= 0; --k) {
    if (seg_off == nullptr) {  // dense bucket totals (chunk-pipelined path)
      XYZZ<F> b = load_xyzz<F>(partials, first + k);
      xyzz_add(run, b);
    } else {
      uint32_t so = __ldg(seg_off + first + k);
      const uint32_t cnt = __ldg(seg_off + first + k + 1) - so;
      if (cnt) {  // non-empty bucket: its total is its first partial (heavy buckets, folded by partial_tree) or the sum of its few runs
        XYZZ<F> b = bucket_total<F>(partials, so, cnt);
        xyzz_add(run, b);
      }
    }
    xyzz_add(acc, run);
  }
  store_xyzz(chunkS, t, run);
  store_xyzz(chunkV, t, acc);
}
// one tree level: node j (multiple of 2*half) absorbs node j+half; the right block starts `half` chunks =
// half*chunk buckets later, so V += V_r + (half*chunk) * S_r  (a power of two: log2 doublings)
template <class F>
__global__ void __launch_bounds__(128) bucket_tree(MsmPlan pl, uint32_t half, uint32_t shift_log2, void* __restrict__ chunkS, void* __restrict__ chunkV) {
  size_t t = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  uint32_t pairs = pl.T / (2 * half);
  if (t >= (size_t)pl.Wr * pairs) return;
  size_t w = t / pairs, j = (t % pairs) * 2 * half;
  size_t left = w * pl.T + j, right = left + half;
  XYZZ<F> Sl = load_xyzz<F>(chunkS, left), Sr = load_xyzz<F>(chunkS, right);
  XYZZ<F> Vl = load_xyzz<F>(chunkV, left), Vr = load_xyzz<F>(chunkV, right);
  xyzz_add(Vl, Vr);
  xyzz_add(Sl, Sr);
  for (uint32_t k = 0; k < shift_log2; ++k) Sr = xyzz_dbl(Sr);
  xyzz_add(Vl, Sr);
  store_xyzz(chunkS, left, Sl);
  store_xyzz(chunkV, left, Vl);
}
// ---- low-latency combination of the chunk results (replaces the pairwise bucket_tree when T >= 64) ------------
// Window total = sum_j A_j + chunk * sum_j j * S_j.  The weighted sum is taken bit by bit:
//   sum_j j * S_j = sum_k 2^k * U_k,   U_k = sum_{j : bit k of j set} S_j
// so every U_k (and the plain sum of the A_j) is an ordinary, perfectly parallel reduction with no doublings in
// it; the only serial part left is one Horner over log2(T) + log2(chunk) doublings.  bucket_tree's pairwise
// merges cost (level + 5) dependent doublings per level, ~90 us each in a lone warp; this is 3 launches.
static constexpr uint32_t kBitParts = 8;      // blocks per (window, bit): each reduces a slice of the chunks
static constexpr uint32_t kBitThreads = 128;
// grid (nbits + 1, Wr, kBitParts); target nbits = plain sum of chunkV
template <class F>
__global__ void __launch_bounds__(kBitThreads) bucket_bitsums(MsmPlan pl, uint32_t nbits, const void* __restrict__ chunkS, const void* __restrict__ chunkV, void* __restrict__ partial) {
  __shared__ uint4 red[kBitThreads * sizeof(XYZZ<F>) / 16];
  const uint32_t k = blockIdx.x, w = blockIdx.y, part = blockIdx.z;
  const uint32_t per = pl.T / kBitParts;  // T >= 64 and a power of two
  XYZZ<F> acc = XYZZ<F>::identity();
  for (uint32_t j = part * per + threadIdx.x; j < (part + 1) * per; j += kBitThreads) {
    if (k == nbits) { XYZZ<F> v = load_xyzz<F>(chunkV, (size_t)w * pl.T + j); xyzz_add(acc, v); }
    else if ((j >> k) & 1) { XYZZ<F> v = load_xyzz<F>(chunkS, (size_t)w * pl.T + j); xyzz_add(acc, v); }
  }
  store_xyzz(red, threadIdx.x, acc);
  __syncthreads();
  for (uint32_t o = kBitThreads / 2; o; o >>= 1) {
    if (threadIdx.x < o) {
      XYZZ<F> a = load_xyzz<F>(red, threadIdx.x), b = load_xyzz<F>(red, threadIdx.x + o);
      xyzz_add(a, b);
      store_xyzz(red, threadIdx.x, a);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) store_xyzz(partial, ((size_t)w * (nbits + 1) + k) * kBitParts + part, load_xyzz<F>(red, 0));
}
// one block per window: thread k folds the kBitParts partials of target k, thread 0 does the Horner and leaves the
// window total where msm_horner expects it (chunkV[w*T])
template <class F>
__global__ void __launch_bounds__(32) bucket_bitfinal(MsmPlan pl, uint32_t nbits, uint32_t chunk_log2, const void* __restrict__ partial, void* __restrict__ chunkV) {
  __shared__ uint4 u[32 * sizeof(XYZZ<F>) / 16];
  const uint32_t w = blockIdx.x, k = threadIdx.x;
  if (k <= nbits) {
    XYZZ<F> acc = XYZZ<F>::identity();
    for (uint32_t part = 0; part < kBitParts; ++part) { XYZZ<F> v = load_xyzz<F>(partial, ((size_t)w * (nbits + 1) + k) * kBitParts + part); xyzz_add(acc, v); }
    store_xyzz(u, k, acc);
  }
  __syncthreads();
  if (k == 0) {
    XYZZ<F> acc = XYZZ<F>::identity();
    for (int b = (int)nbits - 1; b >= 0; --b) { acc = xyzz_dbl(acc); XYZZ<F> v = load_xyzz<F>(u, b); xyzz_add(acc, v); }
    for (uint32_t i = 0; i < chunk_log2; ++i) acc = xyzz_dbl(acc);
    XYZZ<F> a = load_xyzz<F>(u, nbits);
    xyzz_add(acc, a);
    store_xyzz(chunkV, (size_t)w * pl.T, acc);
  }
}

// Horner over the window sums (chunkV[w*T] after the tree): result = sum_w 2^(c*w) * S_w
template <class F>
__global__ void msm_horner(MsmPlan pl, const void* __restrict__ chunkV, void* __restrict__ result) {
  if (blockIdx.x || threadIdx.x) return;
  XYZZ<F> acc = load_xyzz<F>(chunkV, (size_t)(pl.Wr - 1) * pl.T);
  for (int w = (int)pl.Wr - 2; w >= 0; --w) {
    for (uint32_t k = 0; k < pl.c; ++k) acc = xyzz_dbl(acc);
    XYZZ<F> s = load_xyzz<F>(chunkV, (size_t)w * pl.T);
    xyzz_add(acc, s);
  }
  store_xyzz(result, 0, acc);
}
template <class F> __global__ void write_identity(void* result) {
  if (blockIdx.x || threadIdx.x) return;
  store_xyzz(result, 0, XYZZ<F>::identity());
}

// ---- fold partials, normalise, encode ----------------------------------------------------------------------
B2_D void store_be32(uint8_t* out, const Fq& canonical) {
  uint32_t* o = reinterpret_cast<uint32_t*>(out);
#pragma unroll
  for (int k = 0; k < 8; ++k) o[k] = __byte_perm(canonical.v[7 - k], 0, 0x0123);
}
B2_D void encode_point(uint8_t* out, const Affine<Fq>& p, bool native) {
  if (native) { store_affine<Fq>(out, 0, p); return; }
  store_be32(out, Fq::from_mont(p.x)); store_be32(out + 32, Fq::from_mont(p.y));
}
B2_D void encode_point(uint8_t* out, const Affine<Fq2>& p, bool native) {
  if (native) { store_affine<Fq2>(out, 0, p); return; }
  // EIP-197 order x_im | x_re | y_im | y_re (provider.rs:307-320)
  store_be32(out, Fq::from_mont(p.x.c1)); store_be32(out + 32, Fq::from_mont(p.x.c0));
  store_be32(out + 64, Fq::from_mont(p.y.c1)); store_be32(out + 96, Fq::from_mont(p.y.c0));
}
// BLS12-381 G1: native = x | y Montgomery limbs (96 B); else the 48-byte compressed form (big-endian x; bit 7 of byte 0 =
// compressed, bit 6 = infinity, bit 5 = y is the lexicographically larger root) followed by 48 zero bytes, so that the
// [point][is_infinity] layout below keeps the slot size 2 * FieldBytes
B2_D void encode_point(uint8_t* out, const Affine<Fp381>& p, bool native) {
  if (native) { store_affine<Fp381>(out, 0, p); return; }
  uint32_t* o = reinterpret_cast<uint32_t*>(out);
#pragma unroll
  for (int k = 0; k < 24; ++k) o[k] = 0;
  if (p.is_inf()) { out[0] = 0xc0; return; }
  const Fp381 x = Fp381::from_mont(p.x), y = Fp381::from_mont(p.y);
  Fp381 half;
#pragma unroll
  for (int i = 0; i < 12; ++i) half.v[i] = Fp381Cfg::half(i);
#pragma unroll
  for (int k = 0; k < 12; ++k) o[k] = __byte_perm(x.v[11 - k], 0, 0x0123);
  out[0] |= 0x80 | (Fp381::less(half, y) ? 0x20 : 0x00);
}
// d_out layout: [encoded point (64 or 128 B)] [uint32 is_infinity]
template <class F>
__global__ void msm_encode(const void* __restrict__ partials, size_t count, bool native, uint8_t* __restrict__ out) {
  if (blockIdx.x || threadIdx.x) return;
  XYZZ<F> acc = XYZZ<F>::identity();
  for (size_t k = 0; k < count; ++k) { XYZZ<F> p = load_xyzz<F>(partials, k); xyzz_add(acc, p); }
  Affine<F> a = xyzz_to_affine(acc);
  encode_point(out, a, native);
  *reinterpret_cast<uint32_t*>(out + 2 * FieldBytes<F>::value) = a.is_inf() ? 1u : 0u;  // right behind the point: read_result()
}

// ---- Groth16 assembly (b200zk_groth16_fold): fold `count` blocks of partial sums (768 B each: A | B1 | B2 | L | H in
// XYZZ form, one block per rank), normalise and encode.  Four independent single-thread CTAs (each result costs one
// Fermat inversion): 0 -> A, 1 -> B2, 2 -> C = L + H, 3 -> B1.  out: A (64) | B2 (128) | C (64) | B1 (64) | 4 x u32 is_infinity.
__global__ void groth16_assemble(const uint8_t* __restrict__ partials, size_t count, uint8_t* __restrict__ out) {
  if (threadIdx.x) return;
  const uint32_t which = blockIdx.x;
  uint32_t* inf = reinterpret_cast<uint32_t*>(out + 320);
  if (which == 1) {
    XYZZ<Fq2> acc = XYZZ<Fq2>::identity();
    for (size_t k = 0; k < count; ++k) { XYZZ<Fq2> p = load_xyzz<Fq2>(partials + k * 768 + 256, 0); xyzz_add(acc, p); }
    Affine<Fq2> a = xyzz_to_affine(acc);
    encode_point(out + 64, a, false);
    inf[1] = a.is_inf() ? 1u : 0u;
    return;
  }
  XYZZ<Fq> acc = XYZZ<Fq>::identity();
  const size_t off = which == 0 ? 0 : (which == 3 ? 128 : 512);
  for (size_t k = 0; k < count; ++k) {
    XYZZ<Fq> p = load_xyzz<Fq>(partials + k * 768 + off, 0);
    xyzz_add(acc, p);
    if (which == 2) { XYZZ<Fq> h = load_xyzz<Fq>(partials + k * 768 + 640, 0); xyzz_add(acc, h); }
  }
  Affine<Fq> a = xyzz_to_affine(acc);
  encode_point(out + (which == 0 ? 0 : (which == 2 ? 192 : 256)), a, false);
  inf[which == 0 ? 0 : (which == 2 ? 2 : 3)] = a.is_inf() ? 1u : 0u;
}
int groth16_assemble_dev(b200zk_ctx* ctx, const void* d_partials, size_t count, cudaStream_t st, void* d_out) {
  B2_LAUNCH(ctx, groth16_assemble, 4, 32, 0, st, (const uint8_t*)d_partials, count, (uint8_t*)d_out);
  return B200ZK_OK;
}

// ---- zero-knowledge Groth16 assembly (b200zk_groth16_fold_zk): the proof of ark-groth16 0.5 / gnark groth16.Prove for the
// blinding scalars r, s, with the key terms alpha1, beta1, delta1 (g1_terms) and beta2, delta2 (g2_terms) as native affine:
//   A  = alpha1 + [A] + r delta1        B2 = beta2 + [B2] + s delta2        B1 = beta1 + [B1] + s delta1
//   C  = [L] + [H] + s A + r B1 - (rs) delta1
// C is evaluated as [L] + [H] + s (alpha1 + [A]) + r (beta1 + [B1]) + (rs) delta1: the same group element (the r s delta1
// inside s A and inside r B1 cancel against one - rs delta1), but it needs neither A nor B1 first, so the three CTAs
// are independent: 0 -> A (r delta1), 1 -> B2 (s delta2), 2 -> C (one Straus pass over three scalars, 256 shared
// doublings instead of three double-and-add chains).  rs mod r comes from the Fr Montgomery product.  Each CTA ends
// with one Fermat inversion.  out: A (64) | B2 (128) | C (64) | 3 x u32 is_infinity (A, B2, C).
struct G16Blinding {
  uint32_t r[8], s[8];  // canonical little-endian limbs, < the group order
};
B2_D uint32_t scalar_bit(const uint32_t* k, int i) { return (k[i >> 5] >> (i & 31)) & 1u; }
// k * pts[idx] (double-and-add, MSB first) that re-reads the point from memory at every addition instead of keeping
// it live across the loop: those 32 registers are what the Fq2 formulas need to stay clear of local memory
template <class F> B2_D XYZZ<F> scalar_mul_reload(const uint32_t* k, const void* pts, size_t idx) {
  XYZZ<F> acc = XYZZ<F>::identity();
  for (int i = 255; i >= 0; --i) {
    acc = xyzz_dbl(acc);
    if (scalar_bit(k, i)) {
      asm volatile("" ::: "memory");
      const Affine<F> p = load_affine_nc<F>(pts, idx);
      xyzz_add_mixed(acc, p.x, p.y);
    }
  }
  return acc;
}
// acc += *q (add-2008-s, exceptional cases as xyzz_add) for a q parked in shared memory: its coordinates are re-read
// where they are needed instead of being held across the formula, which keeps a G2 addition inside 255 registers
template <class F> B2_D void xyzz_add_parked(XYZZ<F>& acc, const XYZZ<F>* q) {
  if (q->is_inf()) return;
  if (acc.is_inf()) { acc = *q; return; }
  const F U1 = F::mul(acc.x, q->zz), S1 = F::mul(acc.y, q->zzz);
  asm volatile("" ::: "memory");
  const F P = F::sub(F::mul(q->x, acc.zz), U1), R = F::sub(F::mul(q->y, acc.zzz), S1);
  if (P.is_zero()) {
    if (R.is_zero()) acc = xyzz_dbl(acc);
    else acc = XYZZ<F>::identity();
    return;
  }
  const F PP = F::sqr(P), PPP = F::mul(P, PP), Q = F::mul(U1, PP);
  const F x3 = F::sub(F::sub(F::sqr(R), PPP), F::dbl(Q));
  acc.y = F::mul2_sub(R, F::sub(Q, x3), S1, PPP);
  acc.x = x3;
  asm volatile("" ::: "memory");
  acc.zz = F::mul(F::mul(acc.zz, q->zz), PP);
  acc.zzz = F::mul(F::mul(acc.zzz, q->zzz), PPP);
}

// The scalars sit in shared memory (bit lookups with a run-time index stay out of local memory), and every CTA runs its
// scalar multiplication BEFORE folding the partial sums into it, so that no second accumulator is live across the
// 256-step loop.  With scalar_mul_reload and xyzz_add_parked this keeps the G2 branch within 255 registers, no spills.
__global__ void groth16_assemble_zk(const uint8_t* __restrict__ partials, size_t count, const void* __restrict__ g1_terms,
                                    const void* __restrict__ g2_terms, G16Blinding zk, uint8_t* __restrict__ out) {
  __shared__ XYZZ<Fq> table[7];  // Straus table: table[b - 1] = bit0(b) A' + bit1(b) B1' + bit2(b) delta1
  __shared__ uint32_t sc[3][8];  // s, r, rs
  if (threadIdx.x) return;
#pragma unroll
  for (int i = 0; i < 8; ++i) { sc[0][i] = zk.s[i]; sc[1][i] = zk.r[i]; }
  uint32_t* inf = reinterpret_cast<uint32_t*>(out + 256);
  if (blockIdx.x == 1) {  // B2 = s delta2 + beta2 + [B2]
    XYZZ<Fq2> acc = scalar_mul_reload<Fq2>(sc[0], g2_terms, 1);
    const Affine<Fq2> beta = load_affine_nc<Fq2>(g2_terms, 0);
    xyzz_add_mixed(acc, beta.x, beta.y);
    XYZZ<Fq2>* parked = reinterpret_cast<XYZZ<Fq2>*>(table);  // this CTA does not use the Straus table
    for (size_t k = 0; k < count; ++k) {
      *parked = load_xyzz<Fq2>(partials + k * 768 + 256, 0);
      asm volatile("" ::: "memory");
      xyzz_add_parked(acc, parked);
    }
    Affine<Fq2> a = xyzz_to_affine(acc);
    encode_point(out + 64, a, false);
    inf[1] = a.is_inf() ? 1u : 0u;
    return;
  }
  const Affine<Fq> alpha = load_affine_nc<Fq>(g1_terms, 0), delta = load_affine_nc<Fq>(g1_terms, 2);
  if (blockIdx.x == 0) {  // A = r delta1 + alpha1 + [A]
    XYZZ<Fq> a = xyzz_scalar_mul<Fq>(sc[1], delta);
    xyzz_add_mixed(a, alpha.x, alpha.y);
    for (size_t k = 0; k < count; ++k) { XYZZ<Fq> p = load_xyzz<Fq>(partials + k * 768, 0); xyzz_add(a, p); }
    Affine<Fq> aa = xyzz_to_affine(a);
    encode_point(out, aa, false);
    inf[0] = aa.is_inf() ? 1u : 0u;
    return;
  }
  // C = s A' + r B1' + (rs) delta1 + [L] + [H],  A' = alpha1 + [A],  B1' = beta1 + [B1]
  {
    const Affine<Fq> beta = load_affine_nc<Fq>(g1_terms, 1);
    XYZZ<Fq> a = XYZZ<Fq>::identity(), b = XYZZ<Fq>::identity();
    for (size_t k = 0; k < count; ++k) {
      XYZZ<Fq> p = load_xyzz<Fq>(partials + k * 768, 0); xyzz_add(a, p);
      XYZZ<Fq> q = load_xyzz<Fq>(partials + k * 768 + 128, 0); xyzz_add(b, q);
    }
    xyzz_add_mixed(a, alpha.x, alpha.y);
    xyzz_add_mixed(b, beta.x, beta.y);
    table[0] = a; table[1] = b;
    xyzz_add(a, b); table[2] = a;
  }
  table[3] = xyzz_from_affine(delta);
  for (int t = 4; t < 7; ++t) { XYZZ<Fq> e = table[t - 4]; xyzz_add_mixed(e, delta.x, delta.y); table[t] = e; }
  {
    Fr r, s;
#pragma unroll
    for (int i = 0; i < 8; ++i) { r.v[i] = zk.r[i]; s.v[i] = zk.s[i]; }
    const Fr rs = Fr::mul(Fr::to_mont(r), s);  // (r R) s / R = r s mod the group order, canonical
#pragma unroll
    for (int i = 0; i < 8; ++i) sc[2][i] = rs.v[i];
  }
  XYZZ<Fq> c = XYZZ<Fq>::identity();
  for (int i = 255; i >= 0; --i) {
    c = xyzz_dbl(c);
    const uint32_t sel = scalar_bit(sc[0], i) | (scalar_bit(sc[1], i) << 1) | (scalar_bit(sc[2], i) << 2);
    if (sel) { XYZZ<Fq> t = table[sel - 1]; xyzz_add(c, t); }
  }
  for (size_t k = 0; k < count; ++k) {
    XYZZ<Fq> l = load_xyzz<Fq>(partials + k * 768 + 512, 0); xyzz_add(c, l);
    XYZZ<Fq> h = load_xyzz<Fq>(partials + k * 768 + 640, 0); xyzz_add(c, h);
  }
  Affine<Fq> cc = xyzz_to_affine(c);
  encode_point(out + 192, cc, false);
  inf[2] = cc.is_inf() ? 1u : 0u;
}
int groth16_assemble_zk_dev(b200zk_ctx* ctx, const void* d_partials, size_t count, const void* d_g1_terms, const void* d_g2_terms,
                            const uint8_t r_le[32], const uint8_t s_le[32], cudaStream_t st, void* d_out) {
  G16Blinding zk;
  for (int i = 0; i < 8; ++i) {
    zk.r[i] = (uint32_t)r_le[4 * i] | (uint32_t)r_le[4 * i + 1] << 8 | (uint32_t)r_le[4 * i + 2] << 16 | (uint32_t)r_le[4 * i + 3] << 24;
    zk.s[i] = (uint32_t)s_le[4 * i] | (uint32_t)s_le[4 * i + 1] << 8 | (uint32_t)s_le[4 * i + 2] << 16 | (uint32_t)s_le[4 * i + 3] << 24;
  }
  B2_LAUNCH(ctx, groth16_assemble_zk, 3, 32, 0, st, (const uint8_t*)d_partials, count, d_g1_terms, d_g2_terms, zk, (uint8_t*)d_out);
  return B200ZK_OK;
}

// ---- host orchestration ---------------------------------------------------------------------------------------
static inline void phase_mark(b200zk_ctx* ctx, int k, cudaStream_t st) {
  if (ctx->profiling) cudaEventRecord(ctx->ev[k], st);
}

// threads of one accumulation wave: G1 one thread per slice, G2 one lane PAIR per slice (msm_accumulate_g2_pair)
template <class F> static size_t resident_slices(const b200zk_ctx* ctx) {
  if (IsFq2<F>::value) return (size_t)ctx->sm_count * 64u * kG2PairBlocks;
  return (size_t)ctx->sm_count * (sizeof(F) > 32 ? 256u : 512u);
}
template <class F>
static int launch_accumulate(b200zk_ctx* ctx, cudaStream_t st, const void* pts, const uint32_t* idx, const uint32_t* offsets, const uint32_t* run_off, uint32_t G, uint32_t L,
                             size_t slices, void* partials, uint32_t* run_bucket) {
  if constexpr (IsFq2<F>::value)
    B2_LAUNCH(ctx, msm_accumulate_g2_pair, (unsigned)((2 * slices + 127) / 128), 128, 0, st, pts, idx, offsets, run_off, G, L, partials, run_bucket);
  else
    B2_LAUNCH(ctx, msm_accumulate<F>, (unsigned)((slices + 127) / 128), 128, 0, st, pts, idx, offsets, run_off, G, L, partials, run_bucket);
  return B200ZK_OK;
}

// exclusive scan of G values (scan_value: counts, or run flags when seg > 0) into out[0..G]; cursor, if given, receives
// out[0..G) as well.  tsum: one word per kScanTile values.
int exclusive_scan(b200zk_ctx* ctx, cudaStream_t st, const uint32_t* in, const uint32_t* aux, size_t G, uint32_t seg, uint32_t* tsum,
                   uint32_t* out, uint32_t* cursor) {
  const size_t tiles = (G + kScanTile - 1) / kScanTile;
  B2_LAUNCH(ctx, scan_tile_sums, (unsigned)tiles, kScanThreads, 0, st, in, aux, G, seg, tsum);
  B2_LAUNCH(ctx, scan_tile_offsets, 1, 1024, 0, st, tsum, tiles);
  B2_LAUNCH(ctx, scan_apply, (unsigned)tiles, kScanThreads, 0, st, in, aux, G, seg, (const uint32_t*)tsum, out, cursor);
  return B200ZK_OK;
}

// scratch sizes of the two-level sort for up to M_max entries
static size_t sort_ctab_bytes(int sm_count) { return (2 * ((size_t)kSortMaxBins * (size_t)sm_count + 1) + kSortMaxBins + 1) * 4; }
static size_t sort_cnt2_bytes(size_t M_max) { return (M_max / kFineSeg + kSortMaxBins + 1) * (size_t)kSortMaxFine * 4; }

// Digit sort of n scalars into ctx->sort: hist[G] = entries per (window,bucket), offsets[G+1] = their exclusive scan,
// idx[M] = the entries in bucket order.  The two-level sort wherever make_sort_plan accepts the size and plan (it leaves
// hist, offsets and idx exactly as the one-pass sort does), the one-pass msm_hist / scan / msm_scatter everywhere else.
// msm_run has sized the workspace for the sort that runs.
static int sort_digits(b200zk_ctx* ctx, const void* d_scalars, size_t n, uint32_t flags, const MsmPlan& pl, cudaStream_t st) {
  SortWorkspace& s = ctx->sort;
  const size_t G = (size_t)pl.Wr * pl.B;
  uint32_t *hist = (uint32_t*)s.hist.p, *offsets = (uint32_t*)s.offsets.p, *tsum = (uint32_t*)s.tsum.p, *idx = (uint32_t*)s.idx.p;
  SortPlan sp;
  if (!make_sort_plan(n, pl, ctx->sm_count, &sp)) {
    B2_CUDA(ctx, cudaMemsetAsync(hist, 0, G * 4, st));
    const unsigned sgrid = (unsigned)std::min<size_t>((n + 255) / 256, (size_t)ctx->sm_count * 8);
    B2_LAUNCH(ctx, msm_hist, sgrid, 256, 0, st, d_scalars, n, flags, pl, hist, (uint32_t*)s.digits.p);
    phase_mark(ctx, 1, st);
    B2_TRY(exclusive_scan(ctx, st, hist, nullptr, G, 0, tsum, offsets, (uint32_t*)s.cursor.p));
    phase_mark(ctx, 2, st);
    const unsigned wgrid = (unsigned)std::min<size_t>((n * (size_t)pl.W + 255) / 256, (size_t)ctx->sm_count * 32);
    B2_LAUNCH(ctx, msm_scatter, wgrid, 256, 0, st, (const uint32_t*)s.digits.p, n, pl, (uint32_t*)s.cursor.p, idx);
    return B200ZK_OK;
  }
  // two-level: ent1 = W*n 8-byte scratch (value | fine key); ctab = cnt[C*NC+1], base[C*NC+1], item_start
  const size_t Gc = (size_t)sp.C * sp.NC;
  uint32_t *cnt = (uint32_t*)s.ctab.p, *base = cnt + Gc + 1, *item_start = base + Gc + 1, *cnt2 = (uint32_t*)s.cnt2.p;
  uint2* ent1 = (uint2*)s.key.p;
  if (!ctx->attr_sort) {
    B2_CUDA(ctx, cudaFuncSetAttribute(msm_sort_coarse, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SortCoarseSmem)));
    B2_CUDA(ctx, cudaFuncSetAttribute(msm_sort_fine_place, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SortFineSmem)));
    ctx->attr_sort = true;
  }
  B2_CUDA(ctx, cudaMemsetAsync(cnt, 0, (Gc + 1) * 4, st));
  B2_LAUNCH(ctx, msm_sort_count, sp.NC * kSortCountSub, kHistTile, 0, st, d_scalars, n, flags, pl, sp, cnt);
  phase_mark(ctx, 1, st);
  B2_TRY(exclusive_scan(ctx, st, cnt, nullptr, Gc, 0, tsum, base));
  phase_mark(ctx, 2, st);
  B2_LAUNCH(ctx, msm_sort_coarse, sp.NC, kSortTile, sizeof(SortCoarseSmem), st, d_scalars, n, flags, pl, sp, (const uint32_t*)base, ent1);
  // fine pass over segments of kFineSeg entries: at most M / kFineSeg + C items (the grid is this bound; surplus CTAs exit)
  const unsigned max_items = (unsigned)((n * (size_t)pl.W) / kFineSeg + sp.C + 1);
  const uint32_t F = 1u << sp.fb;
  B2_LAUNCH(ctx, msm_sort_items, 1, 1024, 0, st, (const uint32_t*)base, sp, item_start);
  B2_LAUNCH(ctx, msm_sort_fine_count, max_items, 1024, 0, st, (const uint2*)ent1, sp, (const uint32_t*)base, (const uint32_t*)item_start, cnt2);
  B2_LAUNCH(ctx, msm_sort_fine_prefix, (unsigned)(((size_t)sp.C * F + 255) / 256), 256, 0, st, sp, (const uint32_t*)item_start, cnt2, hist);
  B2_TRY(exclusive_scan(ctx, st, hist, nullptr, G, 0, tsum, offsets));
  B2_LAUNCH(ctx, msm_sort_fine_place, max_items, 1024, sizeof(SortFineSmem), st, (const uint2*)ent1, sp, (const uint32_t*)base, (const uint32_t*)item_start, (const uint32_t*)cnt2,
            (const uint32_t*)offsets, idx);
  return B200ZK_OK;
}

// Folds the runs of every bucket with more than kDirectRuns of them into its first run.  Worst case every one of
// `entries` lands in one bucket: ceil(entries / L) + 1 runs to fold.
template <class F>
static int fold_runs(b200zk_ctx* ctx, cudaStream_t st, const uint32_t* run_off, const uint32_t* run_bucket, uint32_t G, size_t entries, uint32_t L, size_t S_max, void* partials) {
  const size_t worst = (entries + 1 + L - 1) / L + 1;
  for (size_t stride = 1; stride < worst; stride *= kTreeRadix)
    B2_LAUNCH(ctx, partial_tree<F>, (unsigned)((S_max + 127) / 128), 128, 0, st, run_off, run_bucket, G, (uint32_t)stride, partials);
  return B200ZK_OK;
}

// Bucket reduction and Horner: d_partial = sum_w 2^(c*w) sum_b (b+1) * B[w][b], from the dense totals in ws_totals
// (run_off == nullptr) or from the runs in ws_buckets that run_off numbers.
template <class F>
static int reduce_buckets(b200zk_ctx* ctx, cudaStream_t st, const MsmPlan& pl, const uint32_t* run_off, void* d_partial) {
  const size_t xy = 4 * FieldBytes<F>::value;
  const size_t chunks = (size_t)pl.Wr * pl.T;
  const void* totals = run_off ? ctx->ws_buckets.p : ctx->ws_totals.p;
  B2_LAUNCH(ctx, bucket_chunk<F>, (unsigned)((chunks + 127) / 128), 128, 0, st, totals, run_off, pl, ctx->ws_chunkS.p, ctx->ws_chunkV.p);
  uint32_t chunk_log2 = 0;
  while ((1u << chunk_log2) < pl.chunk) ++chunk_log2;
  if (pl.T >= 64) {
    uint32_t nbits = 0;
    while ((1u << nbits) < pl.T) ++nbits;
    B2_TRY(ensure(ctx, ctx->ws_bitpart, (size_t)pl.Wr * (nbits + 1) * kBitParts * xy));
    B2_LAUNCH(ctx, bucket_bitsums<F>, dim3(nbits + 1, pl.Wr, kBitParts), kBitThreads, 0, st, pl, nbits, (const void*)ctx->ws_chunkS.p, (const void*)ctx->ws_chunkV.p, ctx->ws_bitpart.p);
    B2_LAUNCH(ctx, bucket_bitfinal<F>, pl.Wr, 32, 0, st, pl, nbits, chunk_log2, (const void*)ctx->ws_bitpart.p, ctx->ws_chunkV.p);
  } else {
    for (uint32_t half = 1, lvl = 0; half < pl.T; half <<= 1, ++lvl) {
      size_t pairs = (size_t)pl.Wr * (pl.T / (2 * half));
      B2_LAUNCH(ctx, bucket_tree<F>, (unsigned)((pairs + 127) / 128), 128, 0, st, pl, half, lvl + chunk_log2, ctx->ws_chunkS.p, ctx->ws_chunkV.p);
    }
  }
  phase_mark(ctx, 5, st);
  B2_LAUNCH(ctx, msm_horner<F>, 1, 32, 0, st, pl, ctx->ws_chunkV.p, d_partial);
  phase_mark(ctx, 6, st);
  return B200ZK_OK;
}

// One schedule for every MSM: the points are cut into K >= 1 chunks, and each chunk is sorted, scanned, accumulated and
// its bucket totals folded before the next; one bucket reduction and Horner close the call.
// Host scalars arrive over PCIe (512 MiB at 2^24, a sizeable fraction of the MSM's time).  On the chunked path chunk k's
// scalars upload on the copy stream (ctx->stream_upload) while earlier chunks compute, so that only the FIRST chunk's
// upload is exposed.  Every kernel runs on the caller's stream in the order sort(0), accumulate(0), sort(1), ...: the
// two-level sort's CTAs want whole SMs, so each kernel has the machine to itself and the copy engine works underneath,
// one chunk ahead.  Profiled calls, shared sorts (sort_mode 1 / 2) and tiny inputs run one chunk and stage host scalars
// on the caller's stream.
template <class F>
static int msm_run(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n, uint32_t flags, cudaStream_t st, void* d_partial,
                   uint32_t table_c, size_t table_stride, const void* h_scalars, int sort_mode) {
  NvtxRange nvtx_msm(IsFq2<F>::value ? "b200zk:g2_msm" : (sizeof(F) > 32 ? "b200zk:bls12_381_g1_msm" : "b200zk:g1_msm"));
  // sort_mode (b200zk_msm_multi_resident_device, groth16_commit): 0 = ordinary call; 1 = one chunk, the digit sort stays in
  // ctx->sort; 2 = the sort of the previous call (same scalars, same plan) is reused: only the point-dependent
  // half of the MSM runs (run scan, accumulation, bucket reduction)
  if (n == 0) {
    B2_LAUNCH(ctx, write_identity<F>, 1, 32, 0, st, d_partial);
    return B200ZK_OK;
  }
  if (n >= ((size_t)1 << 31)) return fail(ctx, B200ZK_ERR_UNSUPPORTED, "msm: n must be < 2^31");
  // 128-bit loads and the bulk copies of the scalar tiles need 16-byte aligned device buffers
  if (((uintptr_t)d_points & 15) || ((uintptr_t)d_scalars & 15)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm: device buffers must be 16-byte aligned");
  MsmPlan pl = make_plan(n, table_c ? table_c : ctx->msm_window, ScalarBits<F>::value);
  if (table_c) {
    pl.merged = 1; pl.Wr = 1; pl.table_stride = (uint32_t)table_stride;
    if ((unsigned long long)table_stride * pl.W >= (1ull << 31)) return fail(ctx, B200ZK_ERR_UNSUPPORTED, "msm: precomputed table too large for 31-bit indices");
  }
  if ((unsigned long long)n * pl.W >= (1ull << 32)) return fail(ctx, B200ZK_ERR_UNSUPPORTED, "msm: n * windows must be < 2^32 (shard the MSM)");
  // with scalars already in HBM one chunk: the accumulation fills the SMs, so there is nothing to overlap; host scalars
  // from 2^22 points up: G1 3 chunks, G2 2 (b200zk_set_msm_chunks overrides the count)
  uint32_t K = ctx->msm_chunks ? ctx->msm_chunks : ((h_scalars && n >= ((size_t)1 << 22)) ? (IsFq2<F>::value ? 2u : 3u) : 1u);
  if (K > kMaxPipelineChunks) K = kMaxPipelineChunks;
  const bool chunked = sort_mode == 0 && (K > 1 || h_scalars) && !ctx->profiling && n >= 4096;
  if (!chunked) K = 1;
  const size_t G = (size_t)pl.Wr * pl.B;
  const size_t xy = 4 * FieldBytes<F>::value, pt = 2 * FieldBytes<F>::value;
  // Chunk k covers points [bnd[k], bnd[k+1]).  With HOST scalars the sizes grow geometrically (ratio r): only the first
  // chunk's upload is exposed, and chunk k+1 uploads while chunk k computes -- the kernels are ~3.7x slower per point than
  // the PCIe copy, so a chunk may be ~3x its predecessor and still arrive in time.  Fewer, larger chunks also pay the
  // per-chunk costs (sort launches, wave tails, bucket_merge over all G buckets) fewer times.  Resident scalars: equal chunks.
  size_t bnd[kMaxPipelineChunks + 1];
  uint32_t chunks = 0;
  {
    // G1 ratio 4, G2 ratio 12: the ratio tracks compute time / copy time
    const double r = h_scalars ? (IsFq2<F>::value ? 12.0 : 4.0) : 1.0;
    double tot = 0, w = 1;
    for (uint32_t k = 0; k < K; ++k) { tot += w; w *= r; }
    double cum = 0; w = 1;
    bnd[0] = 0;
    for (uint32_t k = 0; k < K; ++k) {
      cum += w; w *= r;
      size_t hi = (k == K - 1) ? n : std::min(n, (((size_t)((double)n * (cum / tot))) + 1023) & ~(size_t)1023);
      if (hi > bnd[chunks]) bnd[++chunks] = hi;  // empty chunks (tiny n) vanish
    }
  }
  // per chunk: slice length (each chunk fills whole waves of resident threads); over all chunks: the largest run count and
  // the largest entry count of either sort
  const size_t resident = resident_slices<F>(ctx);
  uint32_t Lk[kMaxPipelineChunks];
  size_t S_max = 0, M_two = 0, M_one = 0;
  for (uint32_t k = 0; k < chunks; ++k) {
    const size_t nk = bnd[k + 1] - bnd[k], Mk = nk * pl.W;
    Lk[k] = pick_slice_len(Mk, resident);
    S_max = std::max(S_max, Mk / Lk[k] + 1 + G);
    SortPlan sp;
    size_t& M_sort = make_sort_plan(nk, pl, ctx->sm_count, &sp) ? M_two : M_one;
    M_sort = std::max(M_sort, Mk);
  }
  // Bucket totals first, one thread per bucket (full occupancy, every lane busy), then the running sums over dense totals:
  // bucket_chunk's threads are few (G / chunk) and serial, so every run addition moved out of them shortens the
  // latency-bound tail.  Dense totals also carry the chunked path's buckets from chunk to chunk.  Below 2^14 buckets a
  // one-chunk call lets bucket_chunk sum the runs itself.
  const bool dense_totals = chunked || G >= ((size_t)1 << 14);
  {
    SortWorkspace& s = ctx->sort;
    const size_t tiles = std::max((G + kScanTile - 1) / kScanTile, ((size_t)kSortMaxBins * ctx->sm_count + kScanTile - 1) / kScanTile);
    B2_TRY(ensure(ctx, s.hist, G * 4));
    B2_TRY(ensure(ctx, s.offsets, (G + 1) * 4));
    B2_TRY(ensure(ctx, s.run_off, (G + 1) * 4));
    B2_TRY(ensure(ctx, s.tsum, tiles * 4));
    B2_TRY(ensure(ctx, s.idx, std::max(M_two, M_one) * 4));
    if (M_one) { B2_TRY(ensure(ctx, s.cursor, G * 4)); B2_TRY(ensure(ctx, s.digits, M_one * 4)); }
    if (M_two) { B2_TRY(ensure(ctx, s.key, M_two * 8)); B2_TRY(ensure(ctx, s.ctab, sort_ctab_bytes(ctx->sm_count))); B2_TRY(ensure(ctx, s.cnt2, sort_cnt2_bytes(M_two))); }
  }
  B2_TRY(ensure(ctx, ctx->ws_buckets, S_max * xy));  // run partials (bucket totals after partial_tree)
  B2_TRY(ensure(ctx, ctx->ws_segbucket, S_max * 4));
  if (dense_totals) B2_TRY(ensure(ctx, ctx->ws_totals, G * xy));
  B2_TRY(ensure(ctx, ctx->ws_chunkS, (size_t)pl.Wr * pl.T * xy));
  B2_TRY(ensure(ctx, ctx->ws_chunkV, (size_t)pl.Wr * pl.T * xy));
  const uint8_t* dsc = (const uint8_t*)d_scalars;
  if (h_scalars) {
    B2_TRY(ensure(ctx, ctx->ws_scalars, n * 32 + 32));
    dsc = (const uint8_t*)ctx->ws_scalars.p;
    if (!chunked) {
      B2_CUDA(ctx, cudaMemcpyAsync(ctx->ws_scalars.p, h_scalars, n * 32, cudaMemcpyHostToDevice, st));
    } else {
      // all uploads issued up front on the copy stream (they serialise on the one H2D engine in chunk order); the staging
      // buffer may still be read by the previous call's kernels on `st`, so the copy stream first waits for `st`
      cudaStream_t cs = ctx->stream_upload;
      B2_CUDA(ctx, cudaEventRecord(ctx->ev_in, st));
      B2_CUDA(ctx, cudaStreamWaitEvent(cs, ctx->ev_in, 0));
      for (uint32_t k = 0; k < chunks; ++k) {
        const size_t lo = bnd[k], nk = bnd[k + 1] - lo;
        B2_CUDA(ctx, cudaMemcpyAsync((void*)(dsc + lo * 32), (const uint8_t*)h_scalars + lo * 32, nk * 32, cudaMemcpyHostToDevice, cs));
        B2_CUDA(ctx, cudaEventRecord(ctx->ev_up[k], cs));
      }
    }
  }
  SortWorkspace& s = ctx->sort;
  uint32_t *hist = (uint32_t*)s.hist.p, *offsets = (uint32_t*)s.offsets.p, *tsum = (uint32_t*)s.tsum.p, *run_off = (uint32_t*)s.run_off.p;
  uint32_t* run_bucket = (uint32_t*)ctx->ws_segbucket.p;
  for (uint32_t k = 0; k < chunks; ++k) {
    const size_t lo = bnd[k], nk = bnd[k + 1] - lo;
    const uint32_t L = Lk[k];
    // sort(k) waits for upload k only: with the kernels serialised there is nothing to gain from sorting ahead, and
    // sort(k+1) before accumulate(k) would stall the stream on upload k+1
    if (chunked && h_scalars) B2_CUDA(ctx, cudaStreamWaitEvent(st, ctx->ev_up[k], 0));
    phase_mark(ctx, 0, st);
    nvtxRangePushA("b200zk:msm_sort");
    if (sort_mode == 2) {
      // hist, offsets and idx are the sort the immediately preceding msm_run on this context left in ctx->sort: its
      // callers (groth16_commit's column loop, msm_multi_resident_device) guarantee that call was mode 1 or 2 over the same
      // scalars and the same plan, and mode 1 runs one chunk, so the whole sort is in the workspace
      phase_mark(ctx, 1, st);
      phase_mark(ctx, 2, st);
    } else {
      B2_TRY(sort_digits(ctx, dsc + lo * 32, nk, flags, pl, st));
    }
    nvtxRangePop();
    phase_mark(ctx, 3, st);
    NvtxRange nvtx_acc("b200zk:msm_accumulate+reduce");
    B2_TRY(exclusive_scan(ctx, st, hist, offsets, G, L, tsum, run_off));
    const size_t Mk = nk * pl.W;
    const void* pts = (const uint8_t*)d_points + lo * pt;
    B2_TRY(launch_accumulate<F>(ctx, st, pts, (const uint32_t*)s.idx.p, offsets, (const uint32_t*)run_off, (uint32_t)G, L, (Mk + L - 1) / L, ctx->ws_buckets.p, run_bucket));
    B2_TRY(fold_runs<F>(ctx, st, run_off, run_bucket, (uint32_t)G, pl.merged ? nk * (size_t)pl.W : nk, L, S_max, ctx->ws_buckets.p));
    phase_mark(ctx, 4, st);
    if (dense_totals) B2_LAUNCH(ctx, bucket_merge<F>, (unsigned)((G + 127) / 128), 128, 0, st, (const void*)ctx->ws_buckets.p, (const uint32_t*)run_off, (uint32_t)G, k == 0 ? 1 : 0, ctx->ws_totals.p);
  }
  return reduce_buckets<F>(ctx, st, pl, dense_totals ? nullptr : run_off, d_partial);
}

template <class F>
static int msm_encode_host(b200zk_ctx* ctx, const void* d_partials, size_t count, uint32_t flags, cudaStream_t st, void* d_out) {
  B2_LAUNCH(ctx, msm_encode<F>, 1, 32, 0, st, d_partials, count, (flags & B200ZK_OUT_NATIVE) != 0, (uint8_t*)d_out);
  return B200ZK_OK;
}

// table[w * n + i] = 2^(c*w) * P_i as an affine point, w = 0..W-1 (window 0 = the bases themselves).
// One thread per base; one Fermat inversion per (base, window) -- a one-off cost when the proving key is loaded.
template <class F>
__global__ void __launch_bounds__(128) precompute_windows(const void* __restrict__ bases, size_t n, uint32_t c, uint32_t W, void* __restrict__ table) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  Affine<F> p = load_affine_nc<F>(bases, i);
  store_affine<F>(table, i, p);
  for (uint32_t w = 1; w < W; ++w) {
    XYZZ<F> q = xyzz_from_affine(p);
    for (uint32_t k = 0; k < c; ++k) q = xyzz_dbl(q);
    p = xyzz_to_affine(q);
    store_affine<F>(table, (size_t)w * n + i, p);
  }
}
template <class F>
static int precompute_host(b200zk_ctx* ctx, const void* d_bases, size_t n, uint32_t c, void* d_table, cudaStream_t st) {
  const uint32_t W = (ScalarBits<F>::value + c - 1) / c;
  if (n) B2_LAUNCH(ctx, precompute_windows<F>, (unsigned)((n + 127) / 128), 128, 0, st, d_bases, n, c, W, d_table);
  return B200ZK_OK;
}
int msm_precompute_g1(b200zk_ctx* ctx, const void* b, size_t n, uint32_t c, void* t, cudaStream_t st) { return precompute_host<Fq>(ctx, b, n, c, t, st); }
int msm_precompute_g2(b200zk_ctx* ctx, const void* b, size_t n, uint32_t c, void* t, cudaStream_t st) { return precompute_host<Fq2>(ctx, b, n, c, t, st); }

// BN254 scalars are always reduced mod r: an unreduced 256-bit scalar (bit 254 or 255 set) would carry a top-window
// coefficient above 2^(c-1), which the signed-digit recoding cannot represent (its bucket index falls outside the tables)
int msm_run_g1(b200zk_ctx* ctx, const void* p, const void* s, size_t n, uint32_t f, cudaStream_t st, void* out, uint32_t tc, size_t ts, const void* hs, int sort_mode) {
  if (f & B200ZK_SCALARS_RAW) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm: B200ZK_SCALARS_RAW is for BLS12-381 calls only");
  return msm_run<Fq>(ctx, p, s, n, f, st, out, tc, ts, hs, sort_mode);
}
int msm_run_g2(b200zk_ctx* ctx, const void* p, const void* s, size_t n, uint32_t f, cudaStream_t st, void* out, uint32_t tc, size_t ts, const void* hs, int sort_mode) {
  if (f & B200ZK_SCALARS_RAW) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm: B200ZK_SCALARS_RAW is for BLS12-381 calls only");
  return msm_run<Fq2>(ctx, p, s, n, f, st, out, tc, ts, hs, sort_mode);
}
int msm_run_bls(b200zk_ctx* ctx, const void* p, const void* s, size_t n, uint32_t f, cudaStream_t st, void* out, uint32_t tc, size_t ts, const void* hs, int sort_mode) { return msm_run<Fp381>(ctx, p, s, n, f | B200ZK_SCALARS_RAW, st, out, tc, ts, hs, sort_mode); }
int msm_precompute_bls(b200zk_ctx* ctx, const void* b, size_t n, uint32_t c, void* t, cudaStream_t st) { return precompute_host<Fp381>(ctx, b, n, c, t, st); }
int msm_encode_bls(b200zk_ctx* ctx, const void* p, size_t c, uint32_t f, cudaStream_t st, void* out) { return msm_encode_host<Fp381>(ctx, p, c, f, st, out); }
int msm_encode_g1(b200zk_ctx* ctx, const void* p, size_t c, uint32_t f, cudaStream_t st, void* out) { return msm_encode_host<Fq>(ctx, p, c, f, st, out); }
int msm_encode_g2(b200zk_ctx* ctx, const void* p, size_t c, uint32_t f, cudaStream_t st, void* out) { return msm_encode_host<Fq2>(ctx, p, c, f, st, out); }

}  // namespace b200zk
