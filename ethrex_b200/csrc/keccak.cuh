// keccak.cuh -- Keccak-f[1600] and keccak256 (original Keccak padding 0x01, not SHA-3's 0x06), host and device.
// Users: ECRECOVER's address hash (secp256k1.cuh, keccak256_64) and the PLONK Fiat-Shamir transcript (plonk.cu, keccak256
// over a transcript of any length).
#pragma once
#include <cstddef>
#include <cstdint>

#include "field.cuh"

namespace b200zk {

// ---- Keccak-f[1600] ----------------------------------------------------------------------------------------------------------
B2_HD uint64_t rotl64(uint64_t x, int s) { return x << s | x >> (64 - s); }  // 0 < s < 64

B2_HD void keccak_f1600(uint64_t* st) {
  constexpr uint64_t rc[24] = {0x0000000000000001ull, 0x0000000000008082ull, 0x800000000000808aull, 0x8000000080008000ull,
                               0x000000000000808bull, 0x0000000080000001ull, 0x8000000080008081ull, 0x8000000000008009ull,
                               0x000000000000008aull, 0x0000000000000088ull, 0x0000000080008009ull, 0x000000008000000aull,
                               0x000000008000808bull, 0x800000000000008bull, 0x8000000000008089ull, 0x8000000000008003ull,
                               0x8000000000008002ull, 0x8000000000000080ull, 0x000000000000800aull, 0x800000008000000aull,
                               0x8000000080008081ull, 0x8000000000008080ull, 0x0000000080000001ull, 0x8000000080008008ull};
  // rho offsets and pi lane order along the cycle starting at lane 1
  constexpr int rotc[24] = {1, 3, 6, 10, 15, 21, 28, 36, 45, 55, 2, 14, 27, 41, 56, 8, 25, 43, 62, 18, 39, 61, 20, 44};
  constexpr int piln[24] = {10, 7, 11, 17, 18, 3, 5, 16, 8, 21, 24, 4, 15, 23, 19, 13, 12, 2, 20, 14, 22, 9, 6, 1};
#pragma unroll 1
  for (int round = 0; round < 24; ++round) {
    uint64_t bc[5];
#pragma unroll
    for (int i = 0; i < 5; ++i) bc[i] = st[i] ^ st[i + 5] ^ st[i + 10] ^ st[i + 15] ^ st[i + 20];
#pragma unroll
    for (int i = 0; i < 5; ++i) {
      const uint64_t t = bc[(i + 4) % 5] ^ rotl64(bc[(i + 1) % 5], 1);
#pragma unroll
      for (int j = 0; j < 25; j += 5) st[j + i] ^= t;
    }
    uint64_t t = st[1];
#pragma unroll
    for (int i = 0; i < 24; ++i) {
      const int j = piln[i];
      const uint64_t u = st[j];
      st[j] = rotl64(t, rotc[i]);
      t = u;
    }
#pragma unroll
    for (int j = 0; j < 25; j += 5) {
#pragma unroll
      for (int i = 0; i < 5; ++i) bc[i] = st[j + i];
#pragma unroll
      for (int i = 0; i < 5; ++i) st[j + i] ^= ~bc[(i + 1) % 5] & bc[(i + 2) % 5];
    }
    st[0] ^= rc[round];
  }
}

// keccak256 of exactly 64 bytes: one absorb (rate 136 bytes), padding 0x01 at byte 64 and 0x80 at byte 135
B2_HD void keccak256_64(const uint8_t* in, uint8_t* out) {
  uint64_t st[25];
#pragma unroll
  for (int i = 0; i < 25; ++i) st[i] = 0;
#pragma unroll
  for (int i = 0; i < 64; ++i) st[i >> 3] |= (uint64_t)in[i] << (8 * (i & 7));
  st[8] ^= 0x01;
  st[16] ^= 0x8000000000000000ull;
  keccak_f1600(st);
#pragma unroll
  for (int i = 0; i < 32; ++i) out[i] = (uint8_t)(st[i >> 3] >> (8 * (i & 7)));
}

// keccak256 of len bytes: rate-136 blocks absorbed in turn, then the padding 0x01 ... 0x80 in the last block
B2_HD void keccak256(const uint8_t* in, size_t len, uint8_t* out) {
  uint64_t st[25];
  for (int i = 0; i < 25; ++i) st[i] = 0;
  size_t off = 0;
  for (; len - off >= 136; off += 136) {
    for (int i = 0; i < 136; ++i) st[i >> 3] ^= (uint64_t)in[off + i] << (8 * (i & 7));
    keccak_f1600(st);
  }
  const int rest = (int)(len - off);
  for (int i = 0; i < rest; ++i) st[i >> 3] ^= (uint64_t)in[off + i] << (8 * (i & 7));
  st[rest >> 3] ^= (uint64_t)0x01 << (8 * (rest & 7));
  st[16] ^= 0x8000000000000000ull;
  keccak_f1600(st);
  for (int i = 0; i < 32; ++i) out[i] = (uint8_t)(st[i >> 3] >> (8 * (i & 7)));
}

}  // namespace b200zk
