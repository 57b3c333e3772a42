// zkey_parse.cpp -- see zkey_parse.h.  The binfileutils container: 4-byte magic, u32 version, u32 section count, then
// sections of u32 id | u64 size | size bytes in any order.  Every size is checked against what the header implies
// before any pointer is handed out, so a caller may read every range of ZkeyLayout.
#include "zkey_parse.h"

#include <cstdarg>
#include <cstdio>
#include <cstring>

namespace b200zk {

namespace {

uint32_t rd32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
uint64_t rd64(const uint8_t* p) { uint64_t v; memcpy(&v, p, 8); return v; }

int refuse(std::string* err, int status, const char* fmt, ...) __attribute__((format(printf, 3, 4)));
int refuse(std::string* err, int status, const char* fmt, ...) {
  char buf[256];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (err) *err = buf;
  return status;
}

bool equals_le(const uint8_t* p, const uint32_t* limbs) {
  for (int i = 0; i < 8; ++i) if (rd32(p + 4 * i) != limbs[i]) return false;
  return true;
}

struct Section { const uint8_t* p = nullptr; uint64_t size = 0; };

// the container's sections with ids 1..max_id (each at most once); other ids are skipped
int read_container(const uint8_t* data, size_t len, const char* what, const char magic[4], uint32_t version, uint32_t max_id,
                   Section* sec, std::string* err) {
  if (!data && len) return refuse(err, B200ZK_ERR_INVALID_ARG, "%s: null buffer", what);
  if (len < 12) return refuse(err, B200ZK_ERR_INVALID_ARG, "%s: truncated: %zu bytes, the file header takes 12", what, len);
  if (memcmp(data, magic, 4) != 0) return refuse(err, B200ZK_ERR_INVALID_ARG, "%s: magic is not \"%.4s\"", what, magic);
  if (rd32(data + 4) != version) return refuse(err, B200ZK_ERR_UNSUPPORTED, "%s: version %u, expected %u", what, rd32(data + 4), version);
  const uint32_t count = rd32(data + 8);
  size_t off = 12;
  for (uint32_t k = 0; k < count; ++k) {
    if (len - off < 12) return refuse(err, B200ZK_ERR_INVALID_ARG, "%s: truncated: header of section %u of %u at byte %zu runs past the end (%zu bytes)", what, k + 1, count, off, len);
    const uint32_t id = rd32(data + off);
    const uint64_t size = rd64(data + off + 4);
    off += 12;
    if (size > len - off) return refuse(err, B200ZK_ERR_INVALID_ARG, "%s: truncated: section %u declares %llu bytes, %zu remain", what, id, (unsigned long long)size, len - off);
    if (id >= 1 && id <= max_id) {
      if (sec[id].p) return refuse(err, B200ZK_ERR_INVALID_ARG, "%s: section %u appears twice", what, id);
      sec[id].p = data + off;
      sec[id].size = size;
    }
    off += size;
  }
  if (off != len) return refuse(err, B200ZK_ERR_INVALID_ARG, "%s: %zu trailing bytes after the last section", what, len - off);
  for (uint32_t id = 1; id <= max_id; ++id)
    if (!sec[id].p) return refuse(err, B200ZK_ERR_INVALID_ARG, "%s: section %u is missing", what, id);
  return B200ZK_OK;
}

int want_size(std::string* err, const char* what, uint32_t id, const char* name, const Section& s, uint64_t bytes) {
  if (s.size == bytes) return B200ZK_OK;
  return refuse(err, B200ZK_ERR_INVALID_ARG, "%s: section %u (%s) holds %llu bytes, the header implies %llu", what, id, name,
                (unsigned long long)s.size, (unsigned long long)bytes);
}

}  // namespace

int zkey_parse(const uint8_t* data, size_t len, ZkeyLayout* out, std::string* err) {
  static const char* kWhat = "zkey";
  Section s[10];
  int rc = read_container(data, len, kWhat, "zkey", 1, 9, s, err);
  if (rc) return rc;
  // section 1: the protocol
  if (s[1].size != 4) return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 1 (protocol) holds %llu bytes, expected 4", (unsigned long long)s[1].size);
  const uint32_t protocol = rd32(s[1].p);
  if (protocol != 1) return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 1: protocol %u is not Groth16 (1)", protocol);
  // section 2: n8q | q | n8r | r | nVars | nPublic | domainSize | alpha1 beta1 beta2 gamma2 delta1 delta2
  const uint8_t* h = s[2].p;
  const uint64_t hs = s[2].size;
  if (hs < 4) return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 2 (header) is truncated at n8q");
  if (rd32(h) != 32) return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 2: n8q = %u, only 32 (BN254) is supported", rd32(h));
  if (hs < 40) return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 2 (header) is truncated at n8r");
  if (!equals_le(h + 4, kZkeyQ)) return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 2: q is not BN254's base-field prime");
  if (rd32(h + 36) != 32) return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 2: n8r = %u, only 32 (BN254) is supported", rd32(h + 36));
  rc = want_size(err, kWhat, 2, "header", s[2], 660);
  if (rc) return rc;
  if (!equals_le(h + 40, kZkeyR)) return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 2: r is not BN254's group order");
  ZkeyLayout L;
  L.n_vars = rd32(h + 72);
  L.n_public = rd32(h + 76);
  L.domain_size = rd32(h + 80);
  if (L.domain_size == 0 || (L.domain_size & (L.domain_size - 1)))
    return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 2: domainSize %u is not a power of two", L.domain_size);
  while ((1u << L.log_n) < L.domain_size) ++L.log_n;
  if (L.log_n > kZkeyMaxLogN)
    return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 2: domainSize 2^%u: the odd coset needs a 2^%u-th root of unity, Fr has none", L.log_n, L.log_n + 1);
  if ((uint64_t)L.n_public + 1 > L.n_vars)
    return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 2: nPublic %u leaves no room for the constant signal in nVars %u", L.n_public, L.n_vars);
  L.alpha1 = h + 84; L.beta1 = h + 148; L.beta2 = h + 212; L.gamma2 = h + 340; L.delta1 = h + 468; L.delta2 = h + 532;
  // sections 3..9: sizes the header implies
  const uint64_t nv = L.n_vars;
  if ((rc = want_size(err, kWhat, 3, "IC", s[3], 64 * ((uint64_t)L.n_public + 1)))) return rc;
  if (s[4].size < 4) return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 4 (coefficients) is truncated at nCoefs");
  L.n_coefs = rd32(s[4].p);
  if ((rc = want_size(err, kWhat, 4, "coefficients", s[4], 4 + kZkeyCoefBytes * (uint64_t)L.n_coefs))) return rc;
  if ((rc = want_size(err, kWhat, 5, "A", s[5], 64 * nv))) return rc;
  if ((rc = want_size(err, kWhat, 6, "B1", s[6], 64 * nv))) return rc;
  if ((rc = want_size(err, kWhat, 7, "B2", s[7], 128 * nv))) return rc;
  if ((rc = want_size(err, kWhat, 8, "C", s[8], 64 * (nv - L.n_public - 1)))) return rc;
  if ((rc = want_size(err, kWhat, 9, "H", s[9], 64 * (uint64_t)L.domain_size))) return rc;
  L.ic = s[3].p;
  L.coefs = s[4].p + 4;
  L.a = s[5].p; L.b1 = s[6].p; L.b2 = s[7].p; L.c = s[8].p; L.h = s[9].p;
  if (out) *out = L;
  return B200ZK_OK;
}

namespace {

// index of the first of n 32-byte little-endian values >= m, or n
size_t first_not_below(const uint8_t* p, size_t n, const uint32_t* m) {
  for (size_t i = 0; i < n; ++i, p += 32) {
    for (int k = 7; k >= 0; --k) {
      const uint32_t v = rd32(p + 4 * k);
      if (v != m[k]) { if (v > m[k]) return i; break; }
      if (k == 0) return i;  // equal
    }
  }
  return n;
}

}  // namespace

int plonk_zkey_parse(const uint8_t* data, size_t len, PlonkLayout* out, std::string* err) {
  static const char* kWhat = "zkey";
  static const char* kQName[5] = {"Qm", "Ql", "Qr", "Qo", "Qc"};
  static const char* kPointName[9] = {"Qm", "Ql", "Qr", "Qo", "Qc", "S1", "S2", "S3", "X_2"};
  Section s[15];
  int rc = read_container(data, len, kWhat, "zkey", 1, 1, s, err);  // the protocol first: a Groth16 key lacks sections 10..14
  if (rc) return rc;
  if (s[1].size == 4 && rd32(s[1].p) != 2) return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 1: protocol %u is not PLONK (2)", rd32(s[1].p));
  s[1] = Section();
  rc = read_container(data, len, kWhat, "zkey", 1, 14, s, err);
  if (rc) return rc;
  if (s[1].size != 4) return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 1 (protocol) holds %llu bytes, expected 4", (unsigned long long)s[1].size);
  const uint32_t protocol = rd32(s[1].p);
  if (protocol != 2) return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 1: protocol %u is not PLONK (2)", protocol);
  // section 2: n8q | q | n8r | r | nVars | nPublic | domainSize | nAdditions | nConstraints | k1 | k2 | 8 G1 | X_2
  const uint8_t* h = s[2].p;
  const uint64_t hs = s[2].size;
  if (hs < 4) return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 2 (header) is truncated at n8q");
  if (rd32(h) != 32) return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 2: n8q = %u, only 32 (BN254) is supported", rd32(h));
  if (hs < 40) return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 2 (header) is truncated at n8r");
  if (!equals_le(h + 4, kZkeyQ)) return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 2: q is not BN254's base-field prime");
  if (rd32(h + 36) != 32) return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 2: n8r = %u, only 32 (BN254) is supported", rd32(h + 36));
  if ((rc = want_size(err, kWhat, 2, "header", s[2], kPlonkHeaderBytes))) return rc;
  if (!equals_le(h + 40, kZkeyR)) return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 2: r is not BN254's group order");
  PlonkLayout L;
  L.n_vars = rd32(h + 72);
  L.n_public = rd32(h + 76);
  L.domain_size = rd32(h + 80);
  L.n_additions = rd32(h + 84);
  L.n_constraints = rd32(h + 88);
  L.k1 = h + 92;
  L.k2 = h + 124;
  L.points = h + 156;
  const uint64_t n = L.domain_size;
  if (n == 0 || (n & (n - 1))) return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 2: domainSize %u is not a power of two", L.domain_size);
  while ((1u << L.log_n) < n) ++L.log_n;
  if (L.log_n > kPlonkMaxLogN)
    return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 2: domainSize 2^%u: the quotient's transforms of size 4 domainSize need 2^%u-th roots of unity, Fr has none",
                  L.log_n, L.log_n + 2);
  if (L.log_n < kPlonkMinLogN) return refuse(err, B200ZK_ERR_UNSUPPORTED, "zkey: section 2: domainSize %u is below 8", L.domain_size);
  if (L.n_public > L.n_constraints) return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 2: nPublic %u exceeds nConstraints %u", L.n_public, L.n_constraints);
  if (L.n_constraints > n) return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 2: nConstraints %u exceeds domainSize %u", L.n_constraints, L.domain_size);
  if ((uint64_t)L.n_additions + L.n_public + 1 > L.n_vars)
    return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 2: nAdditions %u and nPublic %u leave no room for the constant signal in nVars %u", L.n_additions,
                  L.n_public, L.n_vars);
  if (first_not_below(L.k1, 1, kZkeyR) == 0) return refuse(err, B200ZK_ERR_NOT_IN_FIELD, "zkey: section 2: k1 is >= r");
  if (first_not_below(L.k2, 1, kZkeyR) == 0) return refuse(err, B200ZK_ERR_NOT_IN_FIELD, "zkey: section 2: k2 is >= r");
  size_t bad = first_not_below(L.points, 8 * 2 + 4, kZkeyQ);
  if (bad < 20) return refuse(err, B200ZK_ERR_NOT_IN_FIELD, "zkey: section 2: %s has a coordinate >= q", kPointName[bad < 16 ? bad / 2 : 8]);
  // sections 3..14: sizes the header implies
  const uint64_t ext = 5 * n * 32;  // a polynomial section: n coefficients, then 4n evaluations
  if ((rc = want_size(err, kWhat, 3, "additions", s[3], kPlonkAddBytes * (uint64_t)L.n_additions))) return rc;
  static const char* kMapName[3] = {"A map", "B map", "C map"};
  for (int k = 0; k < 3; ++k)
    if ((rc = want_size(err, kWhat, 4 + k, kMapName[k], s[4 + k], 4 * (uint64_t)L.n_constraints))) return rc;
  for (int k = 0; k < 5; ++k)
    if ((rc = want_size(err, kWhat, 7 + k, kQName[k], s[7 + k], ext))) return rc;
  if ((rc = want_size(err, kWhat, 12, "sigma", s[12], 3 * ext))) return rc;
  // snarkjs's plonk_setup.js writes max(nPublic, 1) Lagrange polynomials (L_1 even without public inputs)
  const uint64_t n_lagrange = L.n_public ? L.n_public : 1;
  if ((rc = want_size(err, kWhat, 13, "Lagrange", s[13], n_lagrange * ext))) return rc;
  if ((rc = want_size(err, kWhat, 14, "PTau", s[14], 64 * (n + 6)))) return rc;
  // the records: operands of addition i are signals < nVars - nAdditions + i (earlier signals only), factors < r
  const uint32_t n_wtns = L.n_vars - L.n_additions;
  for (uint32_t i = 0; i < L.n_additions; ++i) {
    const uint8_t* a = s[3].p + kPlonkAddBytes * i;
    const uint32_t s1 = rd32(a), s2 = rd32(a + 4);
    if (s1 >= n_wtns + i || s2 >= n_wtns + i)
      return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section 3: addition %u reads signal %u, not an earlier signal (< %u)", i, s1 >= n_wtns + i ? s1 : s2, n_wtns + i);
    if (first_not_below(a + 8, 2, kZkeyR) < 2) return refuse(err, B200ZK_ERR_NOT_IN_FIELD, "zkey: section 3: addition %u: a factor is >= r", i);
  }
  for (int k = 0; k < 3; ++k)
    for (uint32_t i = 0; i < L.n_constraints; ++i)
      if (rd32(s[4 + k].p + 4 * (size_t)i) >= L.n_vars)
        return refuse(err, B200ZK_ERR_INVALID_ARG, "zkey: section %d (%s): entry %u is signal %u >= nVars %u", 4 + k, kMapName[k], i, rd32(s[4 + k].p + 4 * (size_t)i), L.n_vars);
  // every Fr value of the polynomial sections < r (the 4n evaluations too, though the loader does not use them)
  struct { int id; const char* name; const uint8_t* p; uint64_t values; } polys[7] = {
      {7, "Qm", s[7].p, 5 * n}, {8, "Ql", s[8].p, 5 * n}, {9, "Qr", s[9].p, 5 * n}, {10, "Qo", s[10].p, 5 * n}, {11, "Qc", s[11].p, 5 * n},
      {12, "sigma", s[12].p, 15 * n}, {13, "Lagrange", s[13].p, 5 * n * n_lagrange}};
  for (const auto& q : polys)
    if ((bad = first_not_below(q.p, q.values, kZkeyR)) < q.values)
      return refuse(err, B200ZK_ERR_NOT_IN_FIELD, "zkey: section %d (%s): value %zu is >= r", q.id, q.name, bad);
  if ((bad = first_not_below(s[14].p, 2 * (n + 6), kZkeyQ)) < 2 * (n + 6))
    return refuse(err, B200ZK_ERR_NOT_IN_FIELD, "zkey: section 14 (PTau): point %zu has a coordinate >= q", bad / 2);
  L.additions = s[3].p;
  for (int k = 0; k < 3; ++k) L.map[k] = s[4 + k].p;
  for (int k = 0; k < 5; ++k) L.q[k] = s[7 + k].p;
  L.sigma = s[12].p;
  L.ptau = s[14].p;
  if (out) *out = L;
  return B200ZK_OK;
}

int wtns_parse(const uint8_t* data, size_t len, uint32_t n_vars, const uint8_t** values, std::string* err) {
  static const char* kWhat = "wtns";
  Section s[3];
  int rc = read_container(data, len, kWhat, "wtns", 2, 2, s, err);
  if (rc) return rc;
  // section 1: n8 | prime | nWitness
  if (s[1].size < 4) return refuse(err, B200ZK_ERR_INVALID_ARG, "wtns: section 1 (header) is truncated at n8");
  if (rd32(s[1].p) != 32) return refuse(err, B200ZK_ERR_UNSUPPORTED, "wtns: section 1: n8 = %u, only 32 (BN254) is supported", rd32(s[1].p));
  if ((rc = want_size(err, kWhat, 1, "header", s[1], 40))) return rc;
  if (!equals_le(s[1].p + 4, kZkeyR)) return refuse(err, B200ZK_ERR_UNSUPPORTED, "wtns: section 1: the prime is not BN254's group order");
  const uint32_t n = rd32(s[1].p + 36);
  if (n != n_vars) return refuse(err, B200ZK_ERR_INVALID_ARG, "wtns: section 1: nWitness %u, the key has nVars %u", n, n_vars);
  if ((rc = want_size(err, kWhat, 2, "values", s[2], 32 * (uint64_t)n))) return rc;
  if (values) *values = s[2].p;
  return B200ZK_OK;
}

int zkey_coef_error(int code, size_t record, std::string* err) {
  static const char* kField[] = {"", "matrix is neither 0 (A) nor 1 (B)", "constraint >= domainSize", "signal >= nVars", "value >= r"};
  return refuse(err, code == ZKEY_COEF_VALUE ? B200ZK_ERR_NOT_IN_FIELD : B200ZK_ERR_INVALID_ARG, "zkey: section 4: record %zu: %s", record,
                kField[code >= 1 && code <= 4 ? code : 0]);
}

}  // namespace b200zk
