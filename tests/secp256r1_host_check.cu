// Host build of ethrex_b200/csrc/secp256r1.cuh for tests/test_secp256r1_host.py: nvcc compiles the same
// __host__ __device__ functions the kernel runs into a CPU program, which answers one request per stdin line (values
// are 32-byte big-endian hex):
//   <f>mul|<f>sqr a [b]      Montgomery product on raw limbs, a b 2^-256 mod m   (f = p for P256Fp, n for P256Fn)
//   <f>add|<f>sub a b        canonical values
//   <f>inv a                 a^-1 mod m of a canonical value (through to_mont / from_mont)
//   mont a | unmont a        P256Fp to_mont / from_mont
//   dbl x y l | mdbl x y     2 (x, y) through xyzz_dbl on (l^2 x, l^3 y, l^2, l^3) / xyzz_mdbl: "<x> <y>" affine, "inf"
//   add x1 y1 x2 y2 l        (x1, y1) + (x2, y2) through xyzz_add, the first point scaled by l: "<x> <y>" or "inf"
//   oncurve x y              affine_on_curve: "1" or "0"
//   gmul d                   p256_g_multiple(d): "<x> <y>"
//   verify <160-byte hex>    p256_verify: "1" or "0"
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../ethrex_b200/csrc/secp256r1.cuh"

using namespace b200zk;

static std::vector<uint8_t> unhex(const std::string& h) {
  std::vector<uint8_t> b(h.size() / 2);
  for (size_t i = 0; i < b.size(); ++i) b[i] = (uint8_t)std::stoul(h.substr(2 * i, 2), nullptr, 16);
  return b;
}
static std::string hex(const uint8_t* b, size_t n) {
  static const char* d = "0123456789abcdef";
  std::string s;
  for (size_t i = 0; i < n; ++i) { s += d[b[i] >> 4]; s += d[b[i] & 15]; }
  return s;
}
template <class F> static F fe(const std::string& h) { F a; secp::load_be256(a.v, unhex(h).data()); return a; }
static std::string fe_hex(const uint32_t* v) { uint8_t b[32]; secp::store_be256(b, v); return hex(b, 32); }
static P256Fp mont(const std::string& h) { return P256Fp::to_mont(fe<P256Fp>(h)); }
static std::string affine_hex(const XYZZ<P256Fp>& p) {
  if (p.is_inf()) return "inf";
  const Affine<P256Fp> a = xyzz_to_affine(p);
  return fe_hex(P256Fp::from_mont(a.x).v) + " " + fe_hex(P256Fp::from_mont(a.y).v);
}
static XYZZ<P256Fp> scaled(const std::string& x, const std::string& y, const std::string& l) {  // (l^2 x, l^3 y, l^2, l^3)
  const P256Fp lm = mont(l), l2 = P256Fp::sqr(lm), l3 = P256Fp::mul(l2, lm);
  return {P256Fp::mul(mont(x), l2), P256Fp::mul(mont(y), l3), l2, l3};
}

template <class F> static bool field_op(const std::string& op, const std::string& a, const std::string& b) {
  if (op == "mul") std::cout << fe_hex(F::mul(fe<F>(a), fe<F>(b)).v);
  else if (op == "sqr") std::cout << fe_hex(F::sqr(fe<F>(a)).v);
  else if (op == "add") std::cout << fe_hex(F::add(fe<F>(a), fe<F>(b)).v);
  else if (op == "sub") std::cout << fe_hex(F::sub(fe<F>(a), fe<F>(b)).v);
  else if (op == "inv") std::cout << fe_hex(F::from_mont(F::inv(F::to_mont(fe<F>(a)))).v);
  else return false;
  return true;
}

int main() {
  std::vector<Affine<P256Fp>> gtab(kSecpGTable);
  for (int d = 1; d <= kSecpGTable; ++d) gtab[d - 1] = p256_g_multiple(d);
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, a, b, c, d, e;
    in >> op >> a >> b >> c >> d >> e;
    if (op.size() > 1 && op[0] == 'p' && field_op<P256Fp>(op.substr(1), a, b)) {
    } else if (op.size() > 1 && op[0] == 'n' && field_op<P256Fn>(op.substr(1), a, b)) {
    } else if (op == "mont") std::cout << fe_hex(mont(a).v);
    else if (op == "unmont") std::cout << fe_hex(P256Fp::from_mont(fe<P256Fp>(a)).v);
    else if (op == "dbl") std::cout << affine_hex(xyzz_dbl(scaled(a, b, c)));
    else if (op == "mdbl") std::cout << affine_hex(xyzz_mdbl(mont(a), mont(b)));
    else if (op == "add") {
      XYZZ<P256Fp> acc = scaled(a, b, e);
      xyzz_add(acc, xyzz_from_affine(Affine<P256Fp>{mont(c), mont(d)}));
      std::cout << affine_hex(acc);
    } else if (op == "oncurve") std::cout << (affine_on_curve(Affine<P256Fp>{mont(a), mont(b)}) ? "1" : "0");
    else if (op == "gmul") {
      const Affine<P256Fp> g = p256_g_multiple((uint32_t)std::stoul(a));
      std::cout << fe_hex(P256Fp::from_mont(g.x).v) << " " << fe_hex(P256Fp::from_mont(g.y).v);
    } else if (op == "verify") std::cout << (p256_verify(unhex(a).data(), gtab.data()) ? "1" : "0");
    else std::cout << "? " << op;
    std::cout << "\n";
  }
  return 0;
}
