// pairing.cu -- batched BN254 precompile arithmetic on the GPU: ecAdd, ecMul and the ecPairing check, i.e. the three
// BN254 calls of the reference's `Crypto` trait (/root/reference/crates/common/crypto/provider.rs:201-234 add,
// :239-272 mul, :277-330 pairing check) as the levm precompiles use them
// (/root/reference/crates/vm/levm/src/precompiles.rs:692-745, :775-860: coordinates >= p are rejected BEFORE the
// curve call, G2 travels as x_im | x_re | y_im | y_re).  SURVEY.md section 8(f) rank 4: not a throughput target --
// it is the one part of the path whose results the reference's own tests pin (14 ecpairing vectors,
// /root/reference/test/tests/levm/precompile_tests.rs:17-151), and it runs on the same Fq / Fq2 / XYZZ device code
// as the MSM, so passing those vectors pins that code to the reference directly.
//
// One thread works on one item (a point pair, or one pairing of a check); a batch fills the machine.
// Pairing: PLAIN ate pairing f_{T,Q}(P), T = t - 1 = 6x^2 (127 bits, no Frobenius correction lines), affine line
// functions on the D-type twist (x', y') -> (x' w^2, y' w^3), tower Fq2 = Fq[u]/(u^2+1), Fq6 = Fq2[v]/(v^3 - xi),
// Fq12 = Fq6[w]/(w^2 - v), xi = 9 + u (tower.cuh over Fq2); final exponentiation = conj(f)/f, then one generic power
// (p^6+1)/r.  A
// pairing CHECK asks whether the product is one, which every non-degenerate bilinear pairing on these groups
// answers identically (ark: `Bn254::multi_pairing(..).0 == one`).  oracle/pyref_tower.py is the same algorithm in
// Python; oracle/pyref.py holds an independent optimal-ate statement.
#include "common.cuh"
#include "curve.cuh"
#include "tower.cuh"

namespace b200zk {
namespace {

__constant__ uint32_t kAteT[4] = {0xe87cfd46u, 0xf83e9682u, 0xeeb859fbu, 0x6f4d8248u};  // 6x^2, x = 4965661367192848881
static constexpr int kAteBits = 127;
__constant__ uint32_t kFinalExp[40] = {  // (p^6 + 1) / r, 1268 bits
    0x36e3f812u, 0x5250a540u, 0x96789051u, 0xa5635f15u, 0x4d5bd1d4u, 0xd1138bf5u, 0xbe36c7a2u, 0xa8ce2533u, 0x84e09bf6u, 0x94f69f6bu,
    0x50ef3644u, 0x42ad1f5eu, 0x48c3454cu, 0x0fcc420eu, 0xecc9952cu, 0x758e4408u, 0x87c6042cu, 0xc901bf18u, 0xb14bb3b5u, 0xa733cd65u,
    0xcf51b0d8u, 0xdf6d76bdu, 0x82eb59e1u, 0xca64c0fdu, 0xe39276a1u, 0x1d2e5726u, 0xa391cae9u, 0xc2d1ea74u, 0xc82d647eu, 0x07409206u,
    0xa5afdd17u, 0x051c6d1au, 0x19667af5u, 0xb37f6019u, 0x5084015bu, 0x150e578cu, 0xc23998e4u, 0xfbdea556u, 0xc52f5b83u, 0x000fd14cu};
static constexpr int kFinalExpBits = 1268;

typedef Fp12<Fq2> Fq12;
typedef TowerF2<Fq2> M2;  // the non-inlined Fq2 product and inverse

B2_D Fq2 f2_scale(const Fq2& a, const Fq& k) { return {Fq::mul(a.c0, k), Fq::mul(a.c1, k)}; }

// l(P) = yP - (lam xP) w + (lam xT - yT) w^3, w^3 = v w
B2_D Fq12 line_at(const Fq2& lam, const Fq2& xt, const Fq2& yt, const Affine<Fq>& p) {
  Fq12 l;
  l.c0 = {{p.y, Fq::zero()}, Fq2::zero(), Fq2::zero()};
  l.c1 = {Fq2::neg(f2_scale(lam, p.x)), Fq2::sub(M2::mul(lam, xt), yt), Fq2::zero()};
  return l;
}

// f_{T,Q}(P); neither point is the identity, Q has order r (so no step meets an exceptional case: T < r)
__device__ __noinline__ Fq12 miller_ate(const Affine<Fq2>& q, const Affine<Fq>& p) {
  Fq12 f = Fq12::one();
  Fq2 rx = q.x, ry = q.y;
  for (int i = kAteBits - 2; i >= 0; --i) {
    Fq2 xx = M2::mul(rx, rx);
    Fq2 lam = M2::mul(Fq2::add(Fq2::dbl(xx), xx), M2::inv(Fq2::dbl(ry)));
    f = Fq12::mul(Fq12::mul(f, f), line_at(lam, rx, ry, p));
    Fq2 nx = Fq2::sub(Fq2::sub(M2::mul(lam, lam), rx), rx);
    ry = Fq2::sub(M2::mul(lam, Fq2::sub(rx, nx)), ry);
    rx = nx;
    if ((kAteT[i >> 5] >> (i & 31)) & 1) {
      lam = M2::mul(Fq2::sub(ry, q.y), M2::inv(Fq2::sub(rx, q.x)));
      f = Fq12::mul(f, line_at(lam, rx, ry, p));
      nx = Fq2::sub(Fq2::sub(M2::mul(lam, lam), rx), q.x);
      ry = Fq2::sub(M2::mul(lam, Fq2::sub(rx, nx)), ry);
      rx = nx;
    }
  }
  return f;
}

__device__ __noinline__ Fq12 final_exponentiate(const Fq12& f) {
  Fq12 b = Fq12::mul(Fq12::conj(f), Fq12::inv(f));  // f^(p^6 - 1)
  Fq12 acc = Fq12::one();
  for (int i = kFinalExpBits - 1; i >= 0; --i) {
    acc = Fq12::mul(acc, acc);
    if ((kFinalExp[i >> 5] >> (i & 31)) & 1) acc = Fq12::mul(acc, b);
  }
  return acc;
}

// ---- decoding with the precompile's error order: field range first, then the curve ---------------------------
B2_D Fq load_be_fq(const uint8_t* in, bool* in_range) {
  Fq v;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const uint8_t* b = in + 4 * (7 - k);
    v.v[k] = ((uint32_t)b[0] << 24) | ((uint32_t)b[1] << 16) | ((uint32_t)b[2] << 8) | (uint32_t)b[3];
  }
  Fq m = Fq::modulus(), t;
  *in_range = detail::sub8(t.v, v.v, m.v) != 0;
  return v;
}
B2_D void store_be_fq(uint8_t* out, const Fq& canonical) {
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    uint32_t w = canonical.v[7 - k];
    out[4 * k] = (uint8_t)(w >> 24); out[4 * k + 1] = (uint8_t)(w >> 16); out[4 * k + 2] = (uint8_t)(w >> 8); out[4 * k + 3] = (uint8_t)w;
  }
}
// 0 ok, 2 coordinate >= p, 3 not on the curve
B2_D uint32_t decode_g1(const uint8_t* be, Affine<Fq>* out) {
  bool okx, oky;
  Fq x = load_be_fq(be, &okx), y = load_be_fq(be + 32, &oky);
  if (!(okx && oky)) return B200ZK_ERR_NOT_IN_FIELD;
  *out = {Fq::to_mont(x), Fq::to_mont(y)};
  return affine_on_curve(*out) ? 0u : (uint32_t)B200ZK_ERR_NOT_ON_CURVE;
}
B2_D uint32_t decode_g2(const uint8_t* be, Affine<Fq2>* out) {
  bool ok[4];
  Fq xi = load_be_fq(be, &ok[0]), xr = load_be_fq(be + 32, &ok[1]), yi = load_be_fq(be + 64, &ok[2]), yr = load_be_fq(be + 96, &ok[3]);
  if (!(ok[0] && ok[1] && ok[2] && ok[3])) return B200ZK_ERR_NOT_IN_FIELD;
  *out = {{Fq::to_mont(xr), Fq::to_mont(xi)}, {Fq::to_mont(yr), Fq::to_mont(yi)}};
  return affine_on_curve(*out) ? 0u : (uint32_t)B200ZK_ERR_NOT_ON_CURVE;
}
B2_D void encode_g1(uint8_t* out, const Affine<Fq>& p) {
  store_be_fq(out, Fq::from_mont(p.x));
  store_be_fq(out + 32, Fq::from_mont(p.y));
}

__global__ void __launch_bounds__(64) g1_add_batch(const uint8_t* a, const uint8_t* b, size_t count, uint8_t* out, uint8_t* status) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= count) return;
  Affine<Fq> p, q;
  uint32_t sp = decode_g1(a + 64 * i, &p), sq = decode_g1(b + 64 * i, &q);
  // provider.rs parses p1 then p2; the levm wrapper range-checks both before either curve check
  uint32_t s = (sp == B200ZK_ERR_NOT_IN_FIELD || sq == B200ZK_ERR_NOT_IN_FIELD) ? (uint32_t)B200ZK_ERR_NOT_IN_FIELD : (sp ? sp : sq);
  Affine<Fq> r = {Fq::zero(), Fq::zero()};
  if (!s) {
    XYZZ<Fq> acc = xyzz_from_affine(p);
    xyzz_add_mixed(acc, q.x, q.y);
    r = xyzz_to_affine(acc);
    if (r.is_inf()) s = B200ZK_OK_INFINITY;
  }
  encode_g1(out + 64 * i, r);
  status[i] = (uint8_t)s;
}

__global__ void __launch_bounds__(64) g1_mul_batch(const uint8_t* pts, const uint8_t* scalars, size_t count, uint8_t* out, uint8_t* status) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= count) return;
  Affine<Fq> p;
  uint32_t s = decode_g1(pts + 64 * i, &p);
  Affine<Fq> r = {Fq::zero(), Fq::zero()};
  if (!s) {
    // the group has prime order r, so k*P = (k mod r)*P: the 256-bit scalar is used as it comes
    uint32_t k[8];
    const uint8_t* sb = scalars + 32 * i;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint8_t* b = sb + 4 * (7 - j);
      k[j] = ((uint32_t)b[0] << 24) | ((uint32_t)b[1] << 16) | ((uint32_t)b[2] << 8) | (uint32_t)b[3];
    }
    r = xyzz_to_affine(xyzz_scalar_mul<Fq>(k, p));
    if (r.is_inf()) s = B200ZK_OK_INFINITY;
  }
  encode_g1(out + 64 * i, r);
  status[i] = (uint8_t)s;
}

// one thread per (G1, G2) pair: decode, validate, Miller loop.  f[pair] = 1 when either point is the identity.
__global__ void __launch_bounds__(32) pairing_miller(const uint8_t* pairs, size_t n_pairs, Fq12* f, uint8_t* pair_status) {
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
  if (i >= n_pairs) return;
  Affine<Fq> p;
  Affine<Fq2> q;
  uint32_t sp = decode_g1(pairs + 192 * i, &p), sq = decode_g2(pairs + 192 * i + 64, &q);
  uint32_t s = (sp == B200ZK_ERR_NOT_IN_FIELD || sq == B200ZK_ERR_NOT_IN_FIELD) ? (uint32_t)B200ZK_ERR_NOT_IN_FIELD : (sp ? sp : sq);
  if (!s && !q.is_inf() && !in_subgroup<FrCfg::mod>(q)) s = B200ZK_ERR_NOT_ON_CURVE;  // G1 has cofactor 1: on the curve = in the group
  Fq12 r = Fq12::one();
  if (!s && !p.is_inf() && !q.is_inf()) r = miller_ate(q, p);
  f[i] = r;
  pair_status[i] = (uint8_t)s;
}

}  // namespace

int bn254_g1_add_batch(b200zk_ctx* ctx, const uint8_t* a, const uint8_t* b, size_t count, uint8_t* out, uint8_t* status) {
  if (!count) return B200ZK_OK;
  cudaStream_t st = ctx->stream;
  B2_TRY(ensure(ctx, ctx->ws_points, count * 128));
  B2_TRY(ensure(ctx, ctx->ws_misc, count * 65));
  uint8_t* d_in = (uint8_t*)ctx->ws_points.p;
  uint8_t* d_out = (uint8_t*)ctx->ws_misc.p;
  B2_CUDA(ctx, cudaMemcpyAsync(d_in, a, count * 64, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(d_in + count * 64, b, count * 64, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, g1_add_batch, (unsigned)((count + 63) / 64), 64, 0, st, d_in, d_in + count * 64, count, d_out, d_out + count * 64);
  B2_CUDA(ctx, cudaMemcpyAsync(out, d_out, count * 64, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(status, d_out + count * 64, count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

int bn254_g1_mul_batch(b200zk_ctx* ctx, const uint8_t* points, const uint8_t* scalars, size_t count, uint8_t* out, uint8_t* status) {
  if (!count) return B200ZK_OK;
  cudaStream_t st = ctx->stream;
  B2_TRY(ensure(ctx, ctx->ws_points, count * 96));
  B2_TRY(ensure(ctx, ctx->ws_misc, count * 65));
  uint8_t* d_in = (uint8_t*)ctx->ws_points.p;
  uint8_t* d_out = (uint8_t*)ctx->ws_misc.p;
  B2_CUDA(ctx, cudaMemcpyAsync(d_in, points, count * 64, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(d_in + count * 64, scalars, count * 32, cudaMemcpyHostToDevice, st));
  B2_LAUNCH(ctx, g1_mul_batch, (unsigned)((count + 63) / 64), 64, 0, st, d_in, d_in + count * 64, count, d_out, d_out + count * 64);
  B2_CUDA(ctx, cudaMemcpyAsync(out, d_out, count * 64, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(status, d_out + count * 64, count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

int bn254_pairing_check_batch(b200zk_ctx* ctx, const uint8_t* pairs, const uint32_t* pair_offsets, size_t count, uint8_t* result, uint8_t* status) {
  if (!count) return B200ZK_OK;
  B2_TRY(check_offsets(ctx, pair_offsets, count, "pairing_check_batch"));
  const size_t n_pairs = pair_offsets[count];
  cudaStream_t st = ctx->stream;
  uint8_t *in, *pst, *res, *sts;
  Fq12* f;
  uint32_t* offs;
  B2_TRY(carve(ctx, ctx->ws_points, [&](Carve& c) {
    in = c.take<uint8_t>(192 * n_pairs); f = c.take<Fq12>(n_pairs); pst = c.take<uint8_t>(n_pairs);
    offs = c.take<uint32_t>(count + 1); res = c.take<uint8_t>(count); sts = c.take<uint8_t>(count);
  }));
  if (n_pairs) B2_CUDA(ctx, cudaMemcpyAsync(in, pairs, n_pairs * 192, cudaMemcpyHostToDevice, st));
  B2_CUDA(ctx, cudaMemcpyAsync(offs, pair_offsets, (count + 1) * 4, cudaMemcpyHostToDevice, st));
  if (n_pairs) B2_LAUNCH(ctx, pairing_miller, (unsigned)((n_pairs + 31) / 32), 32, 0, st, in, n_pairs, f, pst);
  B2_LAUNCH(ctx, (pairing_check<Fq12, final_exponentiate>), (unsigned)((count + 31) / 32), 32, 0, st, (const Fq12*)f, pst, (const uint32_t*)offs, count, res, sts);
  B2_CUDA(ctx, cudaMemcpyAsync(result, res, count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaMemcpyAsync(status, sts, count, cudaMemcpyDeviceToHost, st));
  B2_CUDA(ctx, cudaStreamSynchronize(st));
  return B200ZK_OK;
}

}  // namespace b200zk
