// zkey_parse.h -- the snarkjs .zkey (Groth16 and PLONK) and .wtns containers, parsed and validated on the host.
//
// Plain C++ with no CUDA types, so that tests can build it into a CPU program.  The one piece the device shares is
// zkey_coef_check, the check of a section-4 coefficient record: the key loader runs it on every record in a kernel
// (zkey.cu), the CPU test runs the same function over its files.  The layouts are stated in include/b200zk.h.
#pragma once
#include <cstddef>
#include <cstdint>
#include <string>

#include "../../include/b200zk.h"

#if defined(__CUDACC__)
#define ZKEY_HD __host__ __device__ __forceinline__
#else
#define ZKEY_HD inline
#endif

namespace b200zk {

// BN254's group order r and base-field prime q, little-endian 32-bit limbs
constexpr uint32_t kZkeyR[8] = {0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
constexpr uint32_t kZkeyQ[8] = {0xd87cfd47u, 0x3c208c16u, 0x6871ca8du, 0x97816a91u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
constexpr size_t kZkeyCoefBytes = 44;  // u32 matrix | u32 constraint | u32 signal | 32-byte value
constexpr uint32_t kZkeyMaxLogN = 27;  // the odd coset needs the 2^(log_n+1)-th root of unity; Fr has roots up to 2^28

// Pointers into the caller's file.  Points are native affine (G1 64 B, G2 128 B), Montgomery little-endian.
struct ZkeyLayout {
  uint32_t n_vars = 0, n_public = 0, domain_size = 0, log_n = 0, n_coefs = 0;
  const uint8_t *alpha1 = nullptr, *beta1 = nullptr, *beta2 = nullptr, *gamma2 = nullptr, *delta1 = nullptr, *delta2 = nullptr;  // section 2
  const uint8_t* ic = nullptr;     // section 3: n_public + 1 G1 points
  const uint8_t* coefs = nullptr;  // section 4, behind its count: n_coefs records of kZkeyCoefBytes
  const uint8_t *a = nullptr, *b1 = nullptr, *b2 = nullptr, *c = nullptr, *h = nullptr;  // sections 5..9
};

// A snarkjs PLONK key (protocol 2).  Points are native affine G1 (64 B) / G2 (128 B), Fr values Montgomery little-endian.
// Every range below has been size-checked, every map entry, addition operand and Fr value range-checked, and every
// coordinate checked < q (the curve check is the loader's, on the device).
struct PlonkLayout {
  uint32_t n_vars = 0, n_public = 0, domain_size = 0, log_n = 0, n_additions = 0, n_constraints = 0;
  const uint8_t *k1 = nullptr, *k2 = nullptr;   // section 2, 32 bytes each
  const uint8_t* points = nullptr;              // section 2: Qm Ql Qr Qo Qc S1 S2 S3 (G1), then X_2 (G2)
  const uint8_t* additions = nullptr;           // section 3: n_additions records of kPlonkAddBytes
  const uint8_t* map[3] = {nullptr, nullptr, nullptr};  // sections 4..6: n_constraints u32 each
  const uint8_t* q[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // sections 7..11: n coefficients, then 4n evaluations
  const uint8_t* sigma = nullptr;               // section 12: S1, S2, S3 in the same form, 5n values apart
  const uint8_t* ptau = nullptr;                // section 14: domainSize + 6 G1 points
};
constexpr size_t kPlonkAddBytes = 72;     // u32 s1 | u32 s2 | f1 | f2 (Montgomery)
constexpr size_t kPlonkHeaderBytes = 796;
constexpr uint32_t kPlonkMaxLogN = 26;    // the coset transforms run at 4 domainSize <= 2^28
constexpr uint32_t kPlonkMinLogN = 3;     // T's 3n + 6 coefficients must fit in 4n

// Returns a B200ZK_* status; on a refusal *err names the section and the field.
int plonk_zkey_parse(const uint8_t* data, size_t len, PlonkLayout* out, std::string* err);
int zkey_parse(const uint8_t* data, size_t len, ZkeyLayout* out, std::string* err);
// The witness of a key with n_vars signals: *values = section 2, n_vars canonical little-endian 32-byte values
// (their range is checked on the device).
int wtns_parse(const uint8_t* data, size_t len, uint32_t n_vars, const uint8_t** values, std::string* err);

// ---- section-4 record check (host and device) -----------------------------------------------------------------------
enum { ZKEY_COEF_OK = 0, ZKEY_COEF_MATRIX, ZKEY_COEF_CONSTRAINT, ZKEY_COEF_SIGNAL, ZKEY_COEF_VALUE };

// w: the record's 11 little-endian words.  The value must be below r: it is coef * R^2 mod r as snarkjs writes it.
ZKEY_HD int zkey_coef_check(const uint32_t* w, uint32_t domain_size, uint32_t n_vars) {
  if (w[0] > 1) return ZKEY_COEF_MATRIX;
  if (w[1] >= domain_size) return ZKEY_COEF_CONSTRAINT;
  if (w[2] >= n_vars) return ZKEY_COEF_SIGNAL;
  const uint32_t r[8] = {0xf0000001u, 0x43e1f593u, 0x79b97091u, 0x2833e848u, 0x8181585du, 0xb85045b6u, 0xe131a029u, 0x30644e72u};
  for (int i = 7; i >= 0; --i)
    if (w[3 + i] != r[i]) return w[3 + i] < r[i] ? ZKEY_COEF_OK : ZKEY_COEF_VALUE;
  return ZKEY_COEF_VALUE;
}
// the status and message of a failed record check (code != ZKEY_COEF_OK)
int zkey_coef_error(int code, size_t record, std::string* err);

}  // namespace b200zk
