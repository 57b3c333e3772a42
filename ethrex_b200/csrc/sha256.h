// sha256.h -- FIPS 180-4 SHA-256 on the host, for the EIP-4844 Fiat-Shamir challenge (bls381.cu).  A blob's challenge
// hashes one 131,152-byte message: about 2,050 compressions in one serial chain, which a CPU core finishes in well under a
// millisecond and a single GPU thread would not.  Portable C++, no link dependency.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cstring>

namespace b200zk {

class Sha256 {
 public:
  void update(const uint8_t* p, size_t n) {
    total_ += n;
    if (fill_) {
      const size_t take = n < 64 - fill_ ? n : 64 - fill_;
      memcpy(buf_ + fill_, p, take);
      fill_ += take; p += take; n -= take;
      if (fill_ < 64) return;
      block(buf_);
      fill_ = 0;
    }
    for (; n >= 64; p += 64, n -= 64) block(p);
    memcpy(buf_, p, n);
    fill_ = n;
  }
  void final(uint8_t out[32]) {
    const uint64_t bits = total_ * 8;
    const uint8_t pad = 0x80;
    const uint8_t zero[64] = {};
    update(&pad, 1);
    update(zero, fill_ <= 56 ? 56 - fill_ : 120 - fill_);
    uint8_t len[8];
    for (int i = 0; i < 8; ++i) len[i] = (uint8_t)(bits >> (56 - 8 * i));
    update(len, 8);
    for (int i = 0; i < 8; ++i)
      for (int k = 0; k < 4; ++k) out[4 * i + k] = (uint8_t)(h_[i] >> (24 - 8 * k));
  }

 private:
  uint32_t h_[8] = {0x6a09e667u, 0xbb67ae85u, 0x3c6ef372u, 0xa54ff53au, 0x510e527fu, 0x9b05688cu, 0x1f83d9abu, 0x5be0cd19u};
  uint8_t buf_[64];
  size_t fill_ = 0;
  uint64_t total_ = 0;

  static uint32_t rotr(uint32_t x, int s) { return (x >> s) | (x << (32 - s)); }
  void block(const uint8_t* p) {
    static const uint32_t K[64] = {
        0x428a2f98u, 0x71374491u, 0xb5c0fbcfu, 0xe9b5dba5u, 0x3956c25bu, 0x59f111f1u, 0x923f82a4u, 0xab1c5ed5u, 0xd807aa98u, 0x12835b01u, 0x243185beu,
        0x550c7dc3u, 0x72be5d74u, 0x80deb1feu, 0x9bdc06a7u, 0xc19bf174u, 0xe49b69c1u, 0xefbe4786u, 0x0fc19dc6u, 0x240ca1ccu, 0x2de92c6fu, 0x4a7484aau,
        0x5cb0a9dcu, 0x76f988dau, 0x983e5152u, 0xa831c66du, 0xb00327c8u, 0xbf597fc7u, 0xc6e00bf3u, 0xd5a79147u, 0x06ca6351u, 0x14292967u, 0x27b70a85u,
        0x2e1b2138u, 0x4d2c6dfcu, 0x53380d13u, 0x650a7354u, 0x766a0abbu, 0x81c2c92eu, 0x92722c85u, 0xa2bfe8a1u, 0xa81a664bu, 0xc24b8b70u, 0xc76c51a3u,
        0xd192e819u, 0xd6990624u, 0xf40e3585u, 0x106aa070u, 0x19a4c116u, 0x1e376c08u, 0x2748774cu, 0x34b0bcb5u, 0x391c0cb3u, 0x4ed8aa4au, 0x5b9cca4fu,
        0x682e6ff3u, 0x748f82eeu, 0x78a5636fu, 0x84c87814u, 0x8cc70208u, 0x90befffau, 0xa4506cebu, 0xbef9a3f7u, 0xc67178f2u};
    uint32_t w[64];
    for (int i = 0; i < 16; ++i) w[i] = (uint32_t)p[4 * i] << 24 | (uint32_t)p[4 * i + 1] << 16 | (uint32_t)p[4 * i + 2] << 8 | p[4 * i + 3];
    for (int i = 16; i < 64; ++i) {
      const uint32_t s0 = rotr(w[i - 15], 7) ^ rotr(w[i - 15], 18) ^ (w[i - 15] >> 3);
      const uint32_t s1 = rotr(w[i - 2], 17) ^ rotr(w[i - 2], 19) ^ (w[i - 2] >> 10);
      w[i] = w[i - 16] + s0 + w[i - 7] + s1;
    }
    uint32_t a = h_[0], b = h_[1], c = h_[2], d = h_[3], e = h_[4], f = h_[5], g = h_[6], h = h_[7];
    for (int i = 0; i < 64; ++i) {
      const uint32_t t1 = h + (rotr(e, 6) ^ rotr(e, 11) ^ rotr(e, 25)) + ((e & f) ^ (~e & g)) + K[i] + w[i];
      const uint32_t t2 = (rotr(a, 2) ^ rotr(a, 13) ^ rotr(a, 22)) + ((a & b) ^ (a & c) ^ (b & c));
      h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
    }
    h_[0] += a; h_[1] += b; h_[2] += c; h_[3] += d; h_[4] += e; h_[5] += f; h_[6] += g; h_[7] += h;
  }
};

}  // namespace b200zk
