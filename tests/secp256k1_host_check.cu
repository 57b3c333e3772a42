// Host build of ethrex_b200/csrc/secp256k1.cuh for tests/test_secp256k1_host.py: nvcc compiles the same
// __host__ __device__ functions the kernel runs into a CPU program, which answers one request per stdin line:
//   mul|sqr|add|sub|inv a [b]   base field (32-byte big-endian hex in, out)
//   sqrt a                      "1 <root>" or "0"
//   nmul a b | ninv a           scalar field, canonical values
//   sponge <pad> <hex>          keccak-f[1600] sponge, rate 136, domain byte <pad> (1 = keccak256, 6 = SHA3-256)
//   keccak64 <hex>              keccak256_64 of exactly 64 bytes
//   recover <flags> <sig> <msg> "<status> <32-byte hex>"
#include <cstdio>
#include <cstring>
#include <iostream>
#include <sstream>
#include <string>
#include <vector>

#include "../ethrex_b200/csrc/secp256k1.cuh"

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
static SecpFp fe(const std::string& h) { SecpFp a; secp::load_be256(a.v, unhex(h).data()); return a; }
static std::string fe_hex(const uint32_t* v) { uint8_t b[32]; secp::store_be256(b, v); return hex(b, 32); }

static std::string sponge(int pad, const std::vector<uint8_t>& msg) {
  uint64_t st[25] = {};
  std::vector<uint8_t> m = msg;
  m.push_back((uint8_t)pad);
  while (m.size() % 136) m.push_back(0);
  m.back() |= 0x80;
  for (size_t off = 0; off < m.size(); off += 136) {
    for (int i = 0; i < 136; ++i) st[i >> 3] ^= (uint64_t)m[off + i] << (8 * (i & 7));
    keccak_f1600(st);
  }
  uint8_t out[32];
  for (int i = 0; i < 32; ++i) out[i] = (uint8_t)(st[i >> 3] >> (8 * (i & 7)));
  return hex(out, 32);
}

int main() {
  std::vector<Affine<SecpFp>> gtab(kSecpGTable);
  for (int d = 1; d <= kSecpGTable; ++d) gtab[d - 1] = secp_g_multiple(d);
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line);
    std::string op, a, b, c;
    in >> op >> a >> b >> c;
    if (op == "mul") std::cout << fe_hex(SecpFp::mul(fe(a), fe(b)).v);
    else if (op == "sqr") std::cout << fe_hex(SecpFp::sqr(fe(a)).v);
    else if (op == "add") std::cout << fe_hex(SecpFp::add(fe(a), fe(b)).v);
    else if (op == "sub") std::cout << fe_hex(SecpFp::sub(fe(a), fe(b)).v);
    else if (op == "inv") std::cout << fe_hex(SecpFp::inv(fe(a)).v);
    else if (op == "sqrt") {
      SecpFp r;
      if (SecpFp::sqrt(fe(a), &r)) std::cout << "1 " << fe_hex(r.v);
      else std::cout << "0";
    } else if (op == "nmul" || op == "ninv") {
      uint32_t out[8];
      const SecpFn x = SecpFn::from_canonical(fe(a).v);
      (op == "nmul" ? SecpFn::mul(x, SecpFn::from_canonical(fe(b).v)) : SecpFn::inv(x)).to_canonical(out);
      std::cout << fe_hex(out);
    } else if (op == "sponge") std::cout << sponge(std::stoi(a), unhex(b == "-" ? "" : b));
    else if (op == "keccak64") {
      uint8_t out[32];
      keccak256_64(unhex(a).data(), out);
      std::cout << hex(out, 32);
    } else if (op == "recover") {
      uint8_t out[32];
      const uint32_t s = secp_recover(unhex(b).data(), unhex(c).data(), (uint32_t)std::stoul(a), gtab.data(), out);
      std::cout << s << " " << hex(out, 32);
    } else {
      std::cout << "? " << op;
    }
    std::cout << "\n";
  }
  return 0;
}
