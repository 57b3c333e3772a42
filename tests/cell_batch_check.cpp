// CPU program of the cell-batch host unit (ethrex_b200/csrc/cell_batch.cpp), run by tests/test_kzg_verify_cells_host.py.
// One request per stdin line: the path of a file holding n (u64 little-endian), then n commitments (48 bytes each), n cell
// indices (u64 little-endian), n cells (2048 bytes each) and n proofs (48 bytes each).  One answer per request:
//   "bad <k>" when cell k is the first whose index is not below 128, else one line
//   "ok unique=<cells> index=<per cell> commit_off=.. by_commit=.. columns=.. column_off=.. by_column=.. r=<64 hex digits>"
// with each list comma-separated (empty when n = 0).
#include <cstdio>
#include <cstring>
#include <fstream>
#include <iostream>
#include <iterator>
#include <string>
#include <vector>

#include "cell_batch.h"

using namespace b200zk;

static std::string join(const std::vector<uint32_t>& v) {
  std::string s;
  for (size_t i = 0; i < v.size(); ++i) s += (i ? "," : "") + std::to_string(v[i]);
  return s;
}

int main() {
  std::string path;
  while (std::getline(std::cin, path)) {
    std::ifstream f(path, std::ios::binary);
    const std::vector<uint8_t> d((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    uint64_t n = 0;
    memcpy(&n, d.data(), 8);
    const uint8_t* commitments = d.data() + 8;
    std::vector<uint64_t> idx(n);
    if (n) memcpy(idx.data(), commitments + 48 * n, 8 * n);
    const uint8_t* cells = commitments + 56 * n;
    const uint8_t* proofs = cells + kBatchCellBytes * n;
    if (d.size() != 8 + (48 + 8 + kBatchCellBytes + 48) * n) {
      std::cout << "error size" << std::endl;
      continue;
    }
    CellBatch b;
    const size_t bad = cell_batch_build(commitments, idx.data(), n, &b);
    if (bad < n) {
      std::cout << "bad " << bad << std::endl;
      continue;
    }
    uint8_t r[32];
    cell_batch_challenge(b, commitments, idx.data(), cells, proofs, r);
    char hex[65];
    for (int i = 0; i < 32; ++i) snprintf(hex + 2 * i, 3, "%02x", r[i]);
    std::cout << "ok unique=" << join(b.unique) << " index=" << join(b.commit_index) << " commit_off=" << join(b.commit_off)
              << " by_commit=" << join(b.by_commit) << " columns=" << join(b.columns) << " column_off=" << join(b.column_off)
              << " by_column=" << join(b.by_column) << " r=" << hex << std::endl;
  }
  return 0;
}
