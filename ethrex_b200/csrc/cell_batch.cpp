// cell_batch.cpp -- see cell_batch.h
#include "cell_batch.h"

#include <cstring>
#include <string>
#include <unordered_map>

#include "sha256.h"

namespace b200zk {

namespace {
// r, the BLS12-381 group order, little-endian 32-bit limbs
constexpr uint32_t kR[8] = {0x00000001u, 0xffffffffu, 0xfffe5bfeu, 0x53bda402u, 0x09a1d805u, 0x3339d808u, 0x299d7d48u, 0x73eda753u};

void put64(uint8_t* o, uint64_t v) {
  for (int k = 0; k < 8; ++k) o[7 - k] = (uint8_t)(v >> (8 * k));
}

// counting sort of 0..n-1 by key[k] < buckets, stable in k: off (buckets + 1 entries) and the sorted cells
void group_by(const std::vector<uint32_t>& key, size_t buckets, std::vector<uint32_t>* off, std::vector<uint32_t>* sorted) {
  off->assign(buckets + 1, 0);
  for (uint32_t k : key) ++(*off)[k + 1];
  for (size_t i = 0; i < buckets; ++i) (*off)[i + 1] += (*off)[i];
  std::vector<uint32_t> next(off->begin(), off->end() - 1);
  sorted->resize(key.size());
  for (size_t k = 0; k < key.size(); ++k) (*sorted)[next[key[k]]++] = (uint32_t)k;
}
}  // namespace

// < 2^256 < 3r: at most two subtractions
void hash_to_bls_field(const uint8_t d[32], uint8_t z_be[32]) {
  uint32_t v[8];
  for (int k = 0; k < 8; ++k) v[k] = (uint32_t)d[31 - 4 * k] | (uint32_t)d[30 - 4 * k] << 8 | (uint32_t)d[29 - 4 * k] << 16 | (uint32_t)d[28 - 4 * k] << 24;
  for (int pass = 0; pass < 2; ++pass) {
    uint32_t s[8];
    uint64_t br = 0;
    for (int k = 0; k < 8; ++k) { const uint64_t x = (uint64_t)v[k] - kR[k] - br; s[k] = (uint32_t)x; br = (x >> 32) & 1u; }
    if (!br) memcpy(v, s, sizeof v);  // v >= r
  }
  for (int k = 0; k < 8; ++k)
    for (int j = 0; j < 4; ++j) z_be[31 - 4 * k - j] = (uint8_t)(v[k] >> (8 * j));
}

size_t cell_batch_build(const uint8_t* commitments, const uint64_t* cell_indices, size_t n, CellBatch* out) {
  for (size_t k = 0; k < n; ++k)
    if (cell_indices[k] >= kBatchCells) return k;
  CellBatch& b = *out;
  b.n = n;
  b.unique.clear();
  b.commit_index.resize(n);
  std::unordered_map<std::string, uint32_t> seen;
  seen.reserve(n);
  for (size_t k = 0; k < n; ++k) {
    const auto it = seen.emplace(std::string((const char*)commitments + 48 * k, 48), (uint32_t)b.unique.size());
    if (it.second) b.unique.push_back((uint32_t)k);
    b.commit_index[k] = it.first->second;
  }
  group_by(b.commit_index, b.unique.size(), &b.commit_off, &b.by_commit);
  std::vector<uint32_t> col(n), off, sorted;
  for (size_t k = 0; k < n; ++k) col[k] = (uint32_t)cell_indices[k];
  group_by(col, kBatchCells, &off, &sorted);
  b.columns.clear();
  b.column_off.assign(1, 0);
  for (uint32_t c = 0; c < kBatchCells; ++c) {
    if (off[c] == off[c + 1]) continue;
    b.columns.push_back(c);
    b.column_off.push_back(off[c + 1]);
  }
  b.by_column = std::move(sorted);
  return n;
}

void cell_batch_challenge(const CellBatch& b, const uint8_t* commitments, const uint64_t* cell_indices, const uint8_t* cells, const uint8_t* proofs,
                          uint8_t r_be[32]) {
  static const uint8_t kDomain[16] = {'R', 'C', 'K', 'Z', 'G', 'C', 'B', 'A', 'T', 'C', 'H', '_', '_', 'V', '1', '_'};
  uint8_t lens[32];
  put64(lens, kBatchBlobN);
  put64(lens + 8, kBatchCellN);
  put64(lens + 16, b.unique.size());
  put64(lens + 24, b.n);
  Sha256 h;
  h.update(kDomain, 16);
  h.update(lens, 32);
  for (uint32_t k : b.unique) h.update(commitments + 48 * (size_t)k, 48);
  for (size_t k = 0; k < b.n; ++k) {
    uint8_t idx[16];
    put64(idx, b.commit_index[k]);
    put64(idx + 8, cell_indices[k]);
    h.update(idx, 16);
    h.update(cells + kBatchCellBytes * k, kBatchCellBytes);
    h.update(proofs + 48 * k, 48);
  }
  uint8_t digest[32];
  h.final(digest);
  hash_to_bls_field(digest, r_be);
}

}  // namespace b200zk
