// capi.cu -- extern "C" surface of libb200zk.so (include/b200zk.h): lifecycle, host-buffer entry points,
// resident bases, device-pointer entry points, multi-GPU partial/fold.  Style follows the in-tree C-ABI
// precedent /root/reference/crates/guest-program/src/crypto/zisk.rs:5-64 (caller-owned buffers, small integer
// status); the trait these calls sit behind is ProverBackend
// (/root/reference/crates/prover/src/backend/mod.rs:81-147).
#include "common.cuh"
#include <cstdlib>
#include <cstring>
#include <new>

using namespace b200zk;

namespace {

template <bool G2> struct Sizes {
  static constexpr Group group = G2 ? Group::Bn254G2 : Group::Bn254G1;
  static constexpr size_t point = G2 ? 128 : 64;     // affine, native or BE
  static constexpr size_t partial = G2 ? 256 : 128;  // XYZZ
};

int read_result(b200zk_ctx* ctx, const void* d_out, size_t bytes, cudaStream_t st, uint8_t* out) {
  // d_out = [encoded point][u32 is_infinity]
  B2_CUDA(ctx, cudaMemcpyAsync(ctx->h_pinned, d_out, bytes + 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  memcpy(out, ctx->h_pinned, bytes);
  uint32_t inf;
  memcpy(&inf, ctx->h_pinned + bytes, 4);
  return inf ? B200ZK_OK_INFINITY : B200ZK_OK;
}

template <bool G2>
int msm_device_async(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n, uint32_t flags, cudaStream_t st, void* d_out,
                     uint32_t table_c = 0, size_t table_stride = 0, const void* h_scalars = nullptr) {
  if (flags & B200ZK_POINTS_BE) return fail(ctx, B200ZK_ERR_INVALID_ARG, "device entry points take native points");
  B2_TRY(ensure(ctx, ctx->ws_result, 256));
  if (G2) { B2_TRY(msm_run_g2(ctx, d_points, d_scalars, n, flags, st, ctx->ws_result.p, table_c, table_stride, h_scalars)); return msm_encode_g2(ctx, ctx->ws_result.p, 1, flags, st, d_out); }
  B2_TRY(msm_run_g1(ctx, d_points, d_scalars, n, flags, st, ctx->ws_result.p, table_c, table_stride, h_scalars));
  return msm_encode_g1(ctx, ctx->ws_result.p, 1, flags, st, d_out);
}

template <bool G2>
int msm_device(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n, uint32_t flags, void* stream, uint8_t* out,
               uint32_t table_c = 0, size_t table_stride = 0, const void* h_scalars = nullptr) {
  if (!ctx || !out || ((!d_points || (!d_scalars && !h_scalars)) && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm: null argument");
  cudaStream_t st = pick_stream(ctx, stream);
  B2_TRY(ensure(ctx, ctx->ws_out, 256));
  B2_TRY(msm_device_async<G2>(ctx, d_points, d_scalars, n, flags, st, ctx->ws_out.p, table_c, table_stride, h_scalars));
  return read_result(ctx, ctx->ws_out.p, Sizes<G2>::point, st, out);
}

// scalars from host memory into ws_scalars
int stage_scalars(b200zk_ctx* ctx, const void* scalars, size_t n, cudaStream_t st) {
  B2_TRY(ensure(ctx, ctx->ws_scalars, n * 32 + 32));
  if (n) B2_CUDA(ctx, cudaMemcpyAsync(ctx->ws_scalars.p, scalars, n * 32, cudaMemcpyHostToDevice, st));
  return B200ZK_OK;
}

template <bool G2>
int upload_points(b200zk_ctx* ctx, const void* points, size_t n, uint32_t flags, cudaStream_t st, void* d_dst, DevBuf* staging) {
  const size_t bytes = n * Sizes<G2>::point;
  if (!n) return B200ZK_OK;
  if (flags & B200ZK_POINTS_BE) {
    B2_TRY(ensure(ctx, *staging, bytes));
    B2_CUDA(ctx, cudaMemcpyAsync(staging->p, points, bytes, cudaMemcpyHostToDevice, st));
    return points_be_to_native(ctx, staging->p, d_dst, n, G2, st);
  }
  B2_CUDA(ctx, cudaMemcpyAsync(d_dst, points, bytes, cudaMemcpyHostToDevice, st));
  return B200ZK_OK;
}

template <bool G2>
int msm_host(b200zk_ctx* ctx, const void* points, const void* scalars, size_t n, uint32_t flags, uint8_t* out) {
  if (!ctx || !out || ((!points || !scalars) && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm: null argument");
  cudaStream_t st = ctx->stream;
  B2_TRY(ensure(ctx, ctx->ws_points, n * Sizes<G2>::point + 32));
  B2_TRY(upload_points<G2>(ctx, points, n, flags, st, ctx->ws_points.p, &ctx->ws_ntt));
  B2_TRY(stage_scalars(ctx, scalars, n, st));
  return msm_device<G2>(ctx, ctx->ws_points.p, ctx->ws_scalars.p, n, flags & ~B200ZK_POINTS_BE, st, out);
}

template <bool G2>
int bases_upload(b200zk_ctx* ctx, const void* points, size_t n, uint32_t flags, uint64_t* handle) {
  if (!ctx || !handle || (!points && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bases_upload: null argument");
  BasesEntry e;
  e.n = n; e.group = Sizes<G2>::group;
  B2_CUDA(ctx, cudaMalloc(&e.d.p, n * Sizes<G2>::point + 32));
  B2_TRY(upload_points<G2>(ctx, points, n, flags, ctx->stream, e.d.p, &ctx->ws_ntt));
  cudaError_t ce = cudaStreamSynchronize(ctx->stream);
  if (ce != cudaSuccess) return fail(ctx, B200ZK_ERR_CUDA, "bases upload", ce);
  return register_bases(ctx, std::move(e), handle);
}

template <bool G2>
int msm_resident(b200zk_ctx* ctx, uint64_t handle, const void* scalars, size_t n, uint32_t flags, uint8_t* out) {
  if (!ctx || !out || (!scalars && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_resident: null argument");
  const BasesEntry* e = find_bases(ctx, handle, Sizes<G2>::group, "msm_resident: unknown handle");
  if (!e) return B200ZK_ERR_INVALID_ARG;
  if (n > e->n) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_resident: n exceeds the resident bases");
  // host scalars go straight into the (chunk-pipelined) schedule: their upload overlaps the previous chunk's work
  return msm_device<G2>(ctx, e->d.p, nullptr, n, flags & ~B200ZK_POINTS_BE, ctx->stream, out, e->table_c, e->n, scalars);
}

template <bool G2>
int msm_resident_device(b200zk_ctx* ctx, uint64_t handle, const void* d_scalars, size_t n, uint32_t flags, void* stream, uint8_t* out) {
  if (!ctx || !out || (!d_scalars && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_resident_device: null argument");
  const BasesEntry* e = find_bases(ctx, handle, Sizes<G2>::group, "msm_resident_device: unknown handle");
  if (!e) return B200ZK_ERR_INVALID_ARG;
  if (n > e->n) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_resident_device: n exceeds the resident bases");
  return msm_device<G2>(ctx, e->d.p, d_scalars, n, flags & ~B200ZK_POINTS_BE, stream, out, e->table_c, e->n);
}

template <bool G2>
int bases_from_device(b200zk_ctx* ctx, const void* d_points, size_t n, void* stream, uint64_t* handle) {
  if (!ctx || !handle || (!d_points && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bases_from_device: null argument");
  BasesEntry e;
  e.n = n; e.group = Sizes<G2>::group;
  cudaStream_t st = pick_stream(ctx, stream);
  B2_CUDA(ctx, cudaMalloc(&e.d.p, n * Sizes<G2>::point + 32));
  cudaError_t ce = n ? cudaMemcpyAsync(e.d.p, d_points, n * Sizes<G2>::point, cudaMemcpyDeviceToDevice, st) : cudaSuccess;
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(st);
  if (ce != cudaSuccess) return fail(ctx, B200ZK_ERR_CUDA, "bases_from_device copy", ce);
  return register_bases(ctx, std::move(e), handle);
}

template <bool G2>
int fold_partials(b200zk_ctx* ctx, const void* d_partials, size_t count, uint32_t flags, void* stream, uint8_t* out) {
  if (!ctx || !out || (!d_partials && count)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "fold_partials: null argument");
  cudaStream_t st = pick_stream(ctx, stream);
  B2_TRY(ensure(ctx, ctx->ws_out, 256));
  if (G2) B2_TRY(msm_encode_g2(ctx, d_partials, count, flags, st, ctx->ws_out.p));
  else B2_TRY(msm_encode_g1(ctx, d_partials, count, flags, st, ctx->ws_out.p));
  return read_result(ctx, ctx->ws_out.p, Sizes<G2>::point, st, out);
}

}  // namespace

extern "C" {

int b200zk_abi_version(void) { return B200ZK_ABI_VERSION; }

int b200zk_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

const char* b200zk_strerror(int status) {
  switch (status) {
    case B200ZK_OK: return "ok";
    case B200ZK_OK_INFINITY: return "ok (result is the point at infinity)";
    case B200ZK_ERR_NOT_IN_FIELD: return "input coordinate not in field";
    case B200ZK_ERR_NOT_ON_CURVE: return "input point not on curve";
    case B200ZK_ERR_INVALID_ARG: return "invalid argument";
    case B200ZK_ERR_CUDA: return "CUDA error";
    case B200ZK_ERR_NO_DEVICE: return "no CUDA device (this library has no CPU fallback)";
    case B200ZK_ERR_OOM: return "out of device memory";
    case B200ZK_ERR_UNSUPPORTED: return "unsupported size or option";
    default: return "unknown status";
  }
}

int b200zk_init(int device, b200zk_ctx** out) {
  if (!out) return B200ZK_ERR_INVALID_ARG;
  *out = nullptr;
  int n = b200zk_device_count();
  if (n <= 0) return B200ZK_ERR_NO_DEVICE;
  if (device < 0 || device >= n) return B200ZK_ERR_INVALID_ARG;
  b200zk_ctx* ctx = new (std::nothrow) b200zk_ctx();
  if (!ctx) return B200ZK_ERR_OOM;
  ctx->device = device;
  DeviceGuard guard(ctx);  // streams, events and every later allocation belong to `device`; the caller's current device is restored
  int cur = -1;
  if (cudaGetDevice(&cur) != cudaSuccess || cur != device) { cudaGetLastError(); delete ctx; return B200ZK_ERR_CUDA; }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) ctx->sm_count = prop.multiProcessorCount;
  if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
      cudaMallocHost((void**)&ctx->h_pinned, 4096) != cudaSuccess) {
    cudaGetLastError();
    delete ctx;
    return B200ZK_ERR_CUDA;
  }
  for (auto& e : ctx->ev) cudaEventCreate(&e);
  for (auto& e : ctx->ev_plonk) cudaEventCreate(&e);
  {
    // The accumulation gathers 64-byte affine points at random: with the default L2 fetch granularity every gather pulls
    // 128 bytes out of HBM, twice the bytes the gather uses.  A 64-byte granularity is
    // all this library's access patterns need (every stream it reads is either contiguous or 64/128-byte records).
    // The limit is a per-device hint; B200ZK_L2_FETCH=0 leaves the device default, 32 / 64 / 128 set it explicitly.
    const char* e = getenv("B200ZK_L2_FETCH");
    const int want = e ? atoi(e) : 64;
    if (want == 32 || want == 64 || want == 128) { if (cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, (size_t)want) != cudaSuccess) cudaGetLastError(); }
  }
  {
    int lo = 0, hi = 0;
    cudaDeviceGetStreamPriorityRange(&lo, &hi);  // hi = numerically lowest = greatest priority
    if (cudaStreamCreateWithPriority(&ctx->stream_upload, cudaStreamNonBlocking, hi) != cudaSuccess) { cudaGetLastError(); b200zk_destroy(ctx); return B200ZK_ERR_CUDA; }
    cudaEventCreateWithFlags(&ctx->ev_in, cudaEventDisableTiming);
    for (auto& e : ctx->ev_up) cudaEventCreateWithFlags(&e, cudaEventDisableTiming);
  }
  *out = ctx;
  return B200ZK_OK;
}

void b200zk_destroy(b200zk_ctx* ctx) {
  if (!ctx) return;
  int prev_device = -1;
  if (cudaGetDevice(&prev_device) != cudaSuccess) { cudaGetLastError(); prev_device = -1; }
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  // the resident bases, the once-built tables and every workspace DevBuf free themselves (here and in `delete ctx`)
  ctx->bases.clear();
  if (ctx->ev_in) cudaEventDestroy(ctx->ev_in);
  for (auto& e : ctx->ev_up) if (e) cudaEventDestroy(e);
  if (ctx->stream_upload) cudaStreamDestroy(ctx->stream_upload);
  for (auto& kv : ctx->twiddles) { cudaFree(kv.second.d); if (kv.second.ready) cudaEventDestroy(kv.second.ready); }
  for (auto& e : ctx->ev) if (e) cudaEventDestroy(e);
  for (auto& e : ctx->ev_plonk) if (e) cudaEventDestroy(e);
  if (ctx->h_pinned) cudaFreeHost(ctx->h_pinned);
  if (ctx->stream) cudaStreamDestroy(ctx->stream);
  const int own = ctx->device;
  delete ctx;
  if (prev_device >= 0 && prev_device != own) cudaSetDevice(prev_device);
}

const char* b200zk_last_error(const b200zk_ctx* ctx) { return ctx ? ctx->last_error.c_str() : "null context"; }
uint64_t b200zk_launch_count(const b200zk_ctx* ctx) { return ctx ? ctx->launches : 0; }
int b200zk_synchronize(b200zk_ctx* ctx) { b200zk::DeviceGuard guard(ctx);
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  B2_CUDA(ctx, cudaDeviceSynchronize());
  return B200ZK_OK;
}
int b200zk_set_msm_window(b200zk_ctx* ctx, uint32_t c) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || (c && (c < 2 || c > 24))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm window must be 0 or 2..24");
  ctx->msm_window = c;
  return B200ZK_OK;
}
int b200zk_set_msm_chunks(b200zk_ctx* ctx, uint32_t chunks) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || chunks > 64) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm chunks must be 0 (automatic) .. 64");
  ctx->msm_chunks = chunks;
  return B200ZK_OK;
}
int b200zk_set_profiling(b200zk_ctx* ctx, int enabled) { b200zk::DeviceGuard guard(ctx);
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  ctx->profiling = enabled != 0;
  return B200ZK_OK;
}
int b200zk_last_msm_phase_ms(b200zk_ctx* ctx, float out_ms[6]) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || !out_ms) return fail(ctx, B200ZK_ERR_INVALID_ARG, "phase_ms: null argument");
  if (!ctx->profiling) return fail(ctx, B200ZK_ERR_INVALID_ARG, "profiling is off");
  B2_CUDA(ctx, cudaEventSynchronize(ctx->ev[6]));
  for (int k = 0; k < 6; ++k) B2_CUDA(ctx, cudaEventElapsedTime(&out_ms[k], ctx->ev[k], ctx->ev[k + 1]));
  return B200ZK_OK;
}

int b200zk_g1_msm(b200zk_ctx* ctx, const void* points, const void* scalars, size_t n, uint32_t flags, uint8_t out[64]) { b200zk::DeviceGuard guard(ctx); return msm_host<false>(ctx, points, scalars, n, flags, out); }
int b200zk_g2_msm(b200zk_ctx* ctx, const void* points, const void* scalars, size_t n, uint32_t flags, uint8_t out[128]) { b200zk::DeviceGuard guard(ctx); return msm_host<true>(ctx, points, scalars, n, flags, out); }

int b200zk_fr_ntt(b200zk_ctx* ctx, void* data, uint32_t log_n, uint32_t flags, const uint8_t* coset_gen) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || !data) return fail(ctx, B200ZK_ERR_INVALID_ARG, "ntt: null argument");
  if (log_n > 28) return fail(ctx, B200ZK_ERR_INVALID_ARG, "ntt: log_n > 28");
  const size_t bytes = ((size_t)1 << log_n) * 32;
  cudaStream_t st = ctx->stream;
  B2_TRY(ensure(ctx, ctx->ws_points, bytes));
  B2_CUDA(ctx, cudaMemcpyAsync(ctx->ws_points.p, data, bytes, cudaMemcpyHostToDevice, st));
  B2_TRY(ntt_run(ctx, ctx->ws_points.p, log_n, flags, coset_gen, st));
  B2_CUDA(ctx, cudaMemcpyAsync(data, ctx->ws_points.p, bytes, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

int b200zk_g1_bases_upload(b200zk_ctx* ctx, const void* points, size_t n, uint32_t flags, uint64_t* handle) { b200zk::DeviceGuard guard(ctx); return bases_upload<false>(ctx, points, n, flags, handle); }
int b200zk_g2_bases_upload(b200zk_ctx* ctx, const void* points, size_t n, uint32_t flags, uint64_t* handle) { b200zk::DeviceGuard guard(ctx); return bases_upload<true>(ctx, points, n, flags, handle); }
int b200zk_g1_bases_from_device(b200zk_ctx* ctx, const void* d_points, size_t n, void* stream, uint64_t* handle) { b200zk::DeviceGuard guard(ctx); return bases_from_device<false>(ctx, d_points, n, stream, handle); }
int b200zk_g2_bases_from_device(b200zk_ctx* ctx, const void* d_points, size_t n, void* stream, uint64_t* handle) { b200zk::DeviceGuard guard(ctx); return bases_from_device<true>(ctx, d_points, n, stream, handle); }
int b200zk_g1_msm_resident_device(b200zk_ctx* ctx, uint64_t handle, const void* d_scalars, size_t n, uint32_t flags, void* stream, uint8_t out[64]) { b200zk::DeviceGuard guard(ctx); return msm_resident_device<false>(ctx, handle, d_scalars, n, flags, stream, out); }
int b200zk_g2_msm_resident_device(b200zk_ctx* ctx, uint64_t handle, const void* d_scalars, size_t n, uint32_t flags, void* stream, uint8_t out[128]) { b200zk::DeviceGuard guard(ctx); return msm_resident_device<true>(ctx, handle, d_scalars, n, flags, stream, out); }

int b200zk_bases_precompute(b200zk_ctx* ctx, uint64_t handle, uint32_t window_bits) { b200zk::DeviceGuard guard(ctx);
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  BasesEntry* found = find_bases(ctx, handle, "bases_precompute: unknown handle");
  if (!found) return B200ZK_ERR_INVALID_ARG;
  if (window_bits && (window_bits < 2 || window_bits > 24)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bases_precompute: window must be 0 or 2..24");
  BasesEntry& e = *found;
  if (e.group == Group::Bls12G2) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bases_precompute: BLS12-381 G2 handles are pairing inputs, not MSM bases");
  if (e.table_c) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bases_precompute: handle already precomputed");
  const uint32_t c = window_bits ? window_bits : precompute_window(e.n);
  const GroupSizes sz = group_sizes(e.group);
  const uint32_t W = (sz.scalar_bits + c - 1) / c;
  const size_t pt = sz.point;
  if ((unsigned long long)e.n * W >= (1ull << 31)) return fail(ctx, B200ZK_ERR_UNSUPPORTED, "bases_precompute: table exceeds 31-bit indices");
  DevBuf table;
  B2_CUDA(ctx, cudaMalloc(&table.p, (size_t)W * e.n * pt + 32));
  int rc = e.group == Group::Bls12G1 ? msm_precompute_bls(ctx, e.d.p, e.n, c, table.p, ctx->stream)
         : e.group == Group::Bn254G2 ? msm_precompute_g2(ctx, e.d.p, e.n, c, table.p, ctx->stream)
                                     : msm_precompute_g1(ctx, e.d.p, e.n, c, table.p, ctx->stream);
  cudaError_t ce = cudaStreamSynchronize(ctx->stream);
  if (rc > B200ZK_OK_INFINITY) return rc;
  if (ce != cudaSuccess) return fail(ctx, B200ZK_ERR_CUDA, "bases_precompute", ce);
  e.d = std::move(table);
  e.table_c = c;
  return B200ZK_OK;
}

int b200zk_bases_free(b200zk_ctx* ctx, uint64_t handle) { b200zk::DeviceGuard guard(ctx);
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  if (!find_bases(ctx, handle, "bases_free: unknown handle")) return B200ZK_ERR_INVALID_ARG;
  B2_CUDA(ctx, cudaDeviceSynchronize());
  ctx->bases.erase(handle);
  return B200ZK_OK;
}
int b200zk_g1_msm_resident(b200zk_ctx* ctx, uint64_t handle, const void* scalars, size_t n, uint32_t flags, uint8_t out[64]) { b200zk::DeviceGuard guard(ctx); return msm_resident<false>(ctx, handle, scalars, n, flags, out); }
int b200zk_g2_msm_resident(b200zk_ctx* ctx, uint64_t handle, const void* scalars, size_t n, uint32_t flags, uint8_t out[128]) { b200zk::DeviceGuard guard(ctx); return msm_resident<true>(ctx, handle, scalars, n, flags, out); }

int b200zk_g1_msm_device(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n, uint32_t flags, void* stream, uint8_t out[64]) { b200zk::DeviceGuard guard(ctx); return msm_device<false>(ctx, d_points, d_scalars, n, flags, stream, out); }
int b200zk_g2_msm_device(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n, uint32_t flags, void* stream, uint8_t out[128]) { b200zk::DeviceGuard guard(ctx); return msm_device<true>(ctx, d_points, d_scalars, n, flags, stream, out); }
int b200zk_g1_msm_device_async(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n, uint32_t flags, void* stream, void* d_out64) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || !d_out64 || ((!d_points || !d_scalars) && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm: null argument");
  // the encoder appends a 4-byte infinity flag: route through ws_out, then copy the point only
  cudaStream_t st = pick_stream(ctx, stream);
  B2_TRY(ensure(ctx, ctx->ws_out, 256));
  B2_TRY(msm_device_async<false>(ctx, d_points, d_scalars, n, flags, st, ctx->ws_out.p));
  B2_CUDA(ctx, cudaMemcpyAsync(d_out64, ctx->ws_out.p, 64 + 4, cudaMemcpyDeviceToDevice, st));  // point | u32 is_infinity
  return B200ZK_OK;
}
int b200zk_g2_msm_device_async(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n, uint32_t flags, void* stream, void* d_out128) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || !d_out128 || ((!d_points || !d_scalars) && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm: null argument");
  cudaStream_t st = pick_stream(ctx, stream);
  B2_TRY(ensure(ctx, ctx->ws_out, 256));
  B2_TRY(msm_device_async<true>(ctx, d_points, d_scalars, n, flags, st, ctx->ws_out.p));
  B2_CUDA(ctx, cudaMemcpyAsync(d_out128, ctx->ws_out.p, 128 + 4, cudaMemcpyDeviceToDevice, st));  // point | u32 is_infinity
  return B200ZK_OK;
}
int b200zk_fr_ntt_device(b200zk_ctx* ctx, void* d_data, uint32_t log_n, uint32_t flags, const uint8_t* coset_gen, void* stream) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || !d_data) return fail(ctx, B200ZK_ERR_INVALID_ARG, "ntt: null argument");
  return ntt_run(ctx, d_data, log_n, flags, coset_gen, pick_stream(ctx, stream));
}

int b200zk_set_ntt_root(b200zk_ctx* ctx, const uint8_t* root_le) {
  if (!ctx) return B200ZK_ERR_INVALID_ARG;
  DeviceGuard guard(ctx);
  return ntt_set_root(ctx, root_le);
}
int b200zk_ntt_root_preset(int preset, uint8_t root_le_out[32]) {
  // canonical little-endian bytes; values recomputed in tests/test_oracle.py from 5^((r-1)/2^28) and 7^((r-1)/2^28)
  static const uint32_t kArk[8] = {0x725b19f0u, 0x9bd61b6eu, 0x41112ed4u, 0x402d111eu, 0x8ef62abcu, 0x00e0a7ebu, 0xa58a7e85u, 0x2a3c09f0u};
  static const uint32_t kHalo2[8] = {0x60c37c9cu, 0xd34f1ed9u, 0xd39329c8u, 0x3215cf6du, 0x3dd31f74u, 0x98865ea9u, 0x166d18b7u, 0x03ddb9f5u};
  if (!root_le_out || (preset != 0 && preset != 1)) return B200ZK_ERR_INVALID_ARG;
  memcpy(root_le_out, preset ? kHalo2 : kArk, 32);
  return B200ZK_OK;
}

int b200zk_g1_msm_partial_device(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n, uint32_t flags, void* stream, void* d_partial128) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || !d_partial128 || ((!d_points || !d_scalars) && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_partial: null argument");
  if (flags & B200ZK_POINTS_BE) return fail(ctx, B200ZK_ERR_INVALID_ARG, "device entry points take native points");
  return msm_run_g1(ctx, d_points, d_scalars, n, flags, pick_stream(ctx, stream), d_partial128);
}
int b200zk_g2_msm_partial_device(b200zk_ctx* ctx, const void* d_points, const void* d_scalars, size_t n, uint32_t flags, void* stream, void* d_partial256) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || !d_partial256 || ((!d_points || !d_scalars) && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_partial: null argument");
  if (flags & B200ZK_POINTS_BE) return fail(ctx, B200ZK_ERR_INVALID_ARG, "device entry points take native points");
  return msm_run_g2(ctx, d_points, d_scalars, n, flags, pick_stream(ctx, stream), d_partial256);
}
int b200zk_g1_msm_partial_resident_device(b200zk_ctx* ctx, uint64_t handle, const void* d_scalars, size_t n, uint32_t flags, void* stream, void* d_partial128) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || !d_partial128 || (!d_scalars && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_partial_resident: null argument");
  const BasesEntry* e = find_bases(ctx, handle, Group::Bn254G1, "msm_partial_resident: unknown handle");
  if (!e) return B200ZK_ERR_INVALID_ARG;
  if (n > e->n) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_partial_resident: n exceeds the resident bases");
  return msm_run_g1(ctx, e->d.p, d_scalars, n, flags & ~B200ZK_POINTS_BE, pick_stream(ctx, stream), d_partial128, e->table_c, e->n);
}
// host (pinned) scalars: their upload is chunk-pipelined with the accumulation; the partial stays on the device
int b200zk_g1_msm_partial_resident(b200zk_ctx* ctx, uint64_t handle, const void* scalars, size_t n, uint32_t flags, void* stream, void* d_partial128) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || !d_partial128 || (!scalars && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_partial_resident: null argument");
  const BasesEntry* e = find_bases(ctx, handle, Group::Bn254G1, "msm_partial_resident: unknown handle");
  if (!e) return B200ZK_ERR_INVALID_ARG;
  if (n > e->n) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_partial_resident: n exceeds the resident bases");
  return msm_run_g1(ctx, e->d.p, nullptr, n, flags & ~B200ZK_POINTS_BE, pick_stream(ctx, stream), d_partial128, e->table_c, e->n, scalars);
}
int b200zk_g2_msm_partial_resident(b200zk_ctx* ctx, uint64_t handle, const void* scalars, size_t n, uint32_t flags, void* stream, void* d_partial256) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || !d_partial256 || (!scalars && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_partial_resident: null argument");
  const BasesEntry* e = find_bases(ctx, handle, Group::Bn254G2, "msm_partial_resident: unknown handle");
  if (!e) return B200ZK_ERR_INVALID_ARG;
  if (n > e->n) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_partial_resident: n exceeds the resident bases");
  return msm_run_g2(ctx, e->d.p, nullptr, n, flags & ~B200ZK_POINTS_BE, pick_stream(ctx, stream), d_partial256, e->table_c, e->n, scalars);
}
int b200zk_g2_msm_partial_resident_device(b200zk_ctx* ctx, uint64_t handle, const void* d_scalars, size_t n, uint32_t flags, void* stream, void* d_partial256) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || !d_partial256 || (!d_scalars && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_partial_resident: null argument");
  const BasesEntry* e = find_bases(ctx, handle, Group::Bn254G2, "msm_partial_resident: unknown handle");
  if (!e) return B200ZK_ERR_INVALID_ARG;
  if (n > e->n) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_partial_resident: n exceeds the resident bases");
  return msm_run_g2(ctx, e->d.p, d_scalars, n, flags & ~B200ZK_POINTS_BE, pick_stream(ctx, stream), d_partial256, e->table_c, e->n);
}
int b200zk_g1_fold_partials_device(b200zk_ctx* ctx, const void* d_partials, size_t count, uint32_t flags, void* stream, uint8_t out[64]) { b200zk::DeviceGuard guard(ctx); return fold_partials<false>(ctx, d_partials, count, flags, stream, out); }
int b200zk_g2_fold_partials_device(b200zk_ctx* ctx, const void* d_partials, size_t count, uint32_t flags, void* stream, uint8_t out[128]) { b200zk::DeviceGuard guard(ctx); return fold_partials<true>(ctx, d_partials, count, flags, stream, out); }

int b200zk_msm_multi_resident_device(b200zk_ctx* ctx, const uint64_t* handles, size_t count, const void* d_scalars, size_t n, uint32_t flags,
                                     void* stream, uint8_t* out, int* status) {
  DeviceGuard guard(ctx);
  if (!ctx || (count && (!handles || !out || !status)) || (!d_scalars && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_multi_resident_device: null argument");
  if (!count) return B200ZK_OK;
  cudaStream_t st = pick_stream(ctx, stream);
  std::vector<const BasesEntry*> cols(count);
  for (size_t i = 0; i < count; ++i) {
    const BasesEntry* e = cols[i] = find_bases(ctx, handles[i], "msm_multi_resident_device: unknown handle");
    if (!e) return B200ZK_ERR_INVALID_ARG;
    if (n > e->n) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_multi_resident_device: n exceeds the resident bases");
    if (e->group != Group::Bn254G1 && e->group != Group::Bn254G2) return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_multi_resident_device: BLS12-381 bases in a BN254 call");
    // one sort serves every column only if they share the plan: same window tables (or none) over the same point count
    if (e->table_c != cols[0]->table_c || (e->table_c && e->n != cols[0]->n))
      return fail(ctx, B200ZK_ERR_INVALID_ARG, "msm_multi_resident_device: handles must share the precomputed window and the point count");
  }
  B2_TRY(ensure(ctx, ctx->ws_result, 256));
  B2_TRY(ensure(ctx, ctx->ws_out, 256));
  for (size_t i = 0; i < count; ++i) {
    const BasesEntry& e = *cols[i];
    const int mode = (n >= 2) ? (i == 0 ? 1 : 2) : 0;  // n < 2: nothing worth sharing, and the tiny plans differ
    const uint32_t f = flags & ~(uint32_t)B200ZK_POINTS_BE;
    int rc;
    if (e.group == Group::Bn254G2) {
      B2_TRY(msm_run_g2(ctx, e.d.p, d_scalars, n, f, st, ctx->ws_result.p, e.table_c, e.n, nullptr, mode));
      B2_TRY(msm_encode_g2(ctx, ctx->ws_result.p, 1, flags, st, ctx->ws_out.p));
      rc = read_result(ctx, ctx->ws_out.p, 128, st, out + 128 * i);
    } else {
      B2_TRY(msm_run_g1(ctx, e.d.p, d_scalars, n, f, st, ctx->ws_result.p, e.table_c, e.n, nullptr, mode));
      B2_TRY(msm_encode_g1(ctx, ctx->ws_result.p, 1, flags, st, ctx->ws_out.p));
      rc = read_result(ctx, ctx->ws_out.p, 64, st, out + 128 * i);
    }
    if (rc > B200ZK_OK_INFINITY) return rc;
    status[i] = rc;
  }
  return B200ZK_OK;
}

int b200zk_bn254_g1_add_batch(b200zk_ctx* ctx, const uint8_t* a, const uint8_t* b, size_t count, uint8_t* out, uint8_t* status) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || (count && (!a || !b || !out || !status))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bn254_g1_add_batch: null argument");
  return bn254_g1_add_batch(ctx, a, b, count, out, status);
}
int b200zk_bn254_g1_mul_batch(b200zk_ctx* ctx, const uint8_t* points, const uint8_t* scalars, size_t count, uint8_t* out, uint8_t* status) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || (count && (!points || !scalars || !out || !status))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bn254_g1_mul_batch: null argument");
  return bn254_g1_mul_batch(ctx, points, scalars, count, out, status);
}
int b200zk_bn254_pairing_check_batch(b200zk_ctx* ctx, const uint8_t* pairs, const uint32_t* pair_offsets, size_t count, uint8_t* result, uint8_t* status) { b200zk::DeviceGuard guard(ctx);
  if (!ctx || (count && (!pair_offsets || !result || !status))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bn254_pairing_check_batch: null argument");
  if (count && pair_offsets[count] && !pairs) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bn254_pairing_check_batch: null pairs");
  return bn254_pairing_check_batch(ctx, pairs, pair_offsets, count, result, status);
}

}  // extern "C"
