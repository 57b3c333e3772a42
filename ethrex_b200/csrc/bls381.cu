// bls381.cu -- BLS12-381 G1 byte formats on the device and the EIP-4844 blob commitment entry points
// (SURVEY.md section 8f row 3):
//   /root/reference/crates/common/crypto/kzg.rs:259-272        blob_to_kzg_commitment_and_proof -> c_kzg blob_to_kzg_commitment
//   /root/reference/crates/common/types/blobs_bundle.rs:90-118 BlobsBundle::create_from_blobs (one commitment per blob)
// A blob is 4096 field elements (32-byte big-endian, each < the BLS12-381 group order r); its commitment is
// sum_i blob[i] * L_i over the trusted setup's 4096 G1 points in Lagrange form (bit-reversed order, as c-kzg stores them),
// returned in the 48-byte compressed format.  The MSM itself is msm.cu instantiated over Fp381 (window tables included).
#include "common.cuh"
#include <cstring>

namespace b200zk {

B2_D Fp381 load_be48(const uint8_t* in, uint32_t clear_top_mask) {
  const uint32_t* w = reinterpret_cast<const uint32_t*>(in);
  Fp381 v;
#pragma unroll
  for (int k = 0; k < 12; ++k) v.v[k] = __byte_perm(__ldg(w + 11 - k), 0, 0x0123);
  v.v[11] &= clear_top_mask;
  return v;
}

// status[0] = first index whose coordinate is >= p, status[1] = first index that is not a curve point or whose flag bits
// are inconsistent (atomicMin; initialised to n by the host)
__global__ void __launch_bounds__(64) bls_g1_decode(const uint8_t* __restrict__ in, void* __restrict__ native, size_t n, int compressed, unsigned long long* status) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint8_t* src = in + i * (compressed ? 48 : 96);
  const uint8_t flags = src[0];
  const bool c_flag = flags & 0x80, inf_flag = flags & 0x40, sign_flag = flags & 0x20;
  Affine<Fp381> pt = {Fp381::zero(), Fp381::zero()};
  bool bad_field = false, bad_point = false;
  Fp381 x = load_be48(src, 0x1fffffffu);
  if (compressed) {
    if (!c_flag) bad_point = true;
    else if (inf_flag) { if (sign_flag || !x.is_zero()) bad_point = true; }
    else {
      if (!Fp381::less(x, Fp381::modulus())) bad_field = true;
      else {
        const Fp381 xm = Fp381::to_mont(x);
        const Fp381 rhs = Fp381::add(Fp381::mul(Fp381::sqr(xm), xm), CurveB<Fp381>::b());
        Fp381 y = Fp381::sqrt_candidate(rhs);
        if (Fp381::sqr(y) != rhs) bad_point = true;  // x^3 + 4 is not a square: no such point
        else {
          Fp381 half;
#pragma unroll
          for (int k = 0; k < 12; ++k) half.v[k] = Fp381Cfg::half(k);
          const bool largest = Fp381::less(half, Fp381::from_mont(y));
          if (largest != sign_flag) y = Fp381::neg(y);
          pt = {xm, y};
        }
      }
    }
  } else {  // uncompressed: x | y big-endian, flag bits must be clear except infinity
    Fp381 y = load_be48(src + 48, 0xffffffffu);
    if (c_flag || sign_flag) bad_point = true;
    else if (inf_flag) { if (!x.is_zero() || !y.is_zero()) bad_point = true; }
    else if (!Fp381::less(x, Fp381::modulus()) || !Fp381::less(y, Fp381::modulus())) bad_field = true;
    else {
      pt = {Fp381::to_mont(x), Fp381::to_mont(y)};
      if (pt.is_inf() || !affine_on_curve(pt)) bad_point = true;
    }
  }
  if (bad_field) atomicMin(status, (unsigned long long)i);
  if (bad_point) atomicMin(status + 1, (unsigned long long)i);
  if (bad_field || bad_point) pt = {Fp381::zero(), Fp381::zero()};
  store_affine<Fp381>(native, i, pt);
}

// first index of a 32-byte scalar (big-endian, or little-endian limbs) that is not below the BLS12-381 group order
__global__ void __launch_bounds__(256) bls_scalar_check(const uint8_t* __restrict__ scalars, size_t n, int big_endian, unsigned long long* bad) {
  const size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t* w = reinterpret_cast<const uint32_t*>(scalars + 32 * i);
  uint64_t br = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint32_t limb = big_endian ? __byte_perm(__ldg(w + 7 - k), 0, 0x0123) : __ldg(w + k);
    const uint64_t d = (uint64_t)limb - bls_r_limb(k) - br;
    br = (d >> 32) & 1u;
  }
  if (!br) atomicMin(bad, (unsigned long long)i);  // no borrow: scalar >= r
}

int bls_points_to_native(b200zk_ctx* ctx, const void* d_in, void* d_native, size_t n, bool compressed, cudaStream_t st) {
  if (!n) return B200ZK_OK;
  B2_TRY(ensure(ctx, ctx->ws_misc, 512));
  unsigned long long* status = (unsigned long long*)((uint8_t*)ctx->ws_misc.p + 256);
  unsigned long long* h = (unsigned long long*)(ctx->h_pinned + 1024);
  h[0] = h[1] = (unsigned long long)n;
  B2_CUDA(ctx, cudaMemcpyAsync(status, h, 16, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, bls_g1_decode, (unsigned)((n + 63) / 64), 64, 0, st, (const uint8_t*)d_in, d_native, n, compressed ? 1 : 0, status);
  B2_CUDA(ctx, cudaMemcpyAsync(h, status, 16, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  if (h[0] < n && h[0] <= h[1]) return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, "bls12-381 point: coordinate >= p");
  if (h[1] < n) return fail(ctx, B200ZK_ERR_NOT_ON_CURVE, "bls12-381 point: not on the curve or malformed flag bits");
  return B200ZK_OK;
}

int bls_scalars_check(b200zk_ctx* ctx, const void* d_scalars, size_t n, bool big_endian, cudaStream_t st, size_t* bad_index) {
  *bad_index = n;
  if (!n) return B200ZK_OK;
  B2_TRY(ensure(ctx, ctx->ws_misc, 512));
  unsigned long long* status = (unsigned long long*)((uint8_t*)ctx->ws_misc.p + 256);
  unsigned long long* h = (unsigned long long*)(ctx->h_pinned + 1024);
  h[0] = (unsigned long long)n;
  B2_CUDA(ctx, cudaMemcpyAsync(status, h, 8, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, bls_scalar_check, (unsigned)((n + 255) / 256), 256, 0, st, (const uint8_t*)d_scalars, n, big_endian ? 1 : 0, status);
  B2_CUDA(ctx, cudaMemcpyAsync(h, status, 8, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  *bad_index = (size_t)h[0];
  return B200ZK_OK;
}

}  // namespace b200zk

using namespace b200zk;

namespace {
int bls_msm_host_scalars(b200zk_ctx* ctx, const BasesEntry& e, const void* scalars, size_t n, uint32_t flags, cudaStream_t st, uint8_t out[48]) {
  // scalars must be canonical field elements of the BLS12-381 scalar field (c-kzg bytes_to_bls_field rejects the rest), in
  // either byte order: the MSM does not reduce them, and a value >= 2^255 would overflow the signed-digit recoding's top window
  B2_TRY(ensure(ctx, ctx->ws_scalars, n * 32 + 32));
  if (n) B2_CUDA(ctx, cudaMemcpyAsync(ctx->ws_scalars.p, scalars, n * 32, cudaMemcpyHostToDevice, st));
  size_t bad = n;
  B2_TRY(bls_scalars_check(ctx, ctx->ws_scalars.p, n, (flags & B200ZK_SCALARS_BE) != 0, st, &bad));
  if (bad < n) return fail(ctx, B200ZK_ERR_NOT_IN_FIELD, "bls12-381 scalar >= the group order");
  B2_TRY(ensure(ctx, ctx->ws_result, 512));
  B2_TRY(ensure(ctx, ctx->ws_out, 512));
  B2_TRY(msm_run_bls(ctx, e.d, ctx->ws_scalars.p, n, flags & (B200ZK_SCALARS_BE | B200ZK_SCALARS_RAW), st, ctx->ws_result.p, e.table_c, e.n));
  B2_TRY(msm_encode_bls(ctx, ctx->ws_result.p, 1, flags, st, ctx->ws_out.p));
  B2_CUDA(ctx, cudaMemcpyAsync(ctx->h_pinned, ctx->ws_out.p, 96 + 4, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  memcpy(out, ctx->h_pinned, 48);
  uint32_t inf;
  memcpy(&inf, ctx->h_pinned + 96, 4);
  return inf ? B200ZK_OK_INFINITY : B200ZK_OK;
}
}  // namespace

extern "C" {

int b200zk_bls12_381_g1_bases_upload(b200zk_ctx* ctx, const void* points, size_t n, uint32_t flags, uint64_t* handle) {
  if (!ctx || !handle || (!points && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bls12_381_g1_bases_upload: null argument");
  DeviceGuard guard(ctx);
  const bool compressed = flags & B200ZK_POINTS_COMPRESSED;
  const size_t in_bytes = n * (compressed ? 48 : 96);
  BasesEntry e;
  e.n = n; e.g2 = false; e.bls = true;
  B2_CUDA(ctx, cudaMalloc(&e.d, n * 96 + 32));
  int rc = ensure(ctx, ctx->ws_ntt, in_bytes + 32);
  cudaError_t ce = cudaSuccess;
  if (rc <= B200ZK_OK_INFINITY && n) ce = cudaMemcpyAsync(ctx->ws_ntt.p, points, in_bytes, cudaMemcpyHostToDevice, ctx->stream);
  if (rc <= B200ZK_OK_INFINITY && ce == cudaSuccess) rc = bls_points_to_native(ctx, ctx->ws_ntt.p, e.d, n, compressed, ctx->stream);
  if (ce == cudaSuccess) ce = cudaStreamSynchronize(ctx->stream);
  if (rc > B200ZK_OK_INFINITY || ce != cudaSuccess) { cudaFree(e.d); return rc > B200ZK_OK_INFINITY ? rc : fail(ctx, B200ZK_ERR_CUDA, "bls bases upload", ce); }
  *handle = ctx->next_handle++;
  ctx->bases[*handle] = e;
  return B200ZK_OK;
}

int b200zk_bls12_381_g1_msm_resident(b200zk_ctx* ctx, uint64_t handle, const void* scalars, size_t n, uint32_t flags, uint8_t out[48]) {
  if (!ctx || !out || (!scalars && n)) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bls12_381_g1_msm_resident: null argument");
  DeviceGuard guard(ctx);
  auto it = ctx->bases.find(handle);
  if (it == ctx->bases.end() || !it->second.bls) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bls12_381_g1_msm_resident: unknown handle");
  if (n > it->second.n) return fail(ctx, B200ZK_ERR_INVALID_ARG, "bls12_381_g1_msm_resident: n exceeds the resident bases");
  return bls_msm_host_scalars(ctx, it->second, scalars, n, flags, ctx->stream, out);
}

int b200zk_kzg_blob_to_commitment(b200zk_ctx* ctx, uint64_t setup_handle, const uint8_t* blobs, size_t n_blobs, uint8_t* commitments) {
  if (!ctx || (n_blobs && (!blobs || !commitments))) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_blob_to_commitment: null argument");
  DeviceGuard guard(ctx);
  auto it = ctx->bases.find(setup_handle);
  if (it == ctx->bases.end() || !it->second.bls) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_blob_to_commitment: unknown setup handle");
  if (it->second.n != 4096) return fail(ctx, B200ZK_ERR_INVALID_ARG, "kzg_blob_to_commitment: the setup must hold FIELD_ELEMENTS_PER_BLOB = 4096 points");
  for (size_t b = 0; b < n_blobs; ++b) {
    int rc = bls_msm_host_scalars(ctx, it->second, blobs + b * 4096 * 32, 4096, B200ZK_SCALARS_BE | B200ZK_SCALARS_RAW, ctx->stream, commitments + 48 * b);
    if (rc > B200ZK_OK_INFINITY) return rc;
  }
  return B200ZK_OK;
}

}  // extern "C"
