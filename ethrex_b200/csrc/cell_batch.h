// cell_batch.h -- the host half of EIP-7594 verify_cell_kzg_proof_batch over arbitrary cells (b200zk_kzg_verify_cells,
// bls_pairing.cu): the cell-index check, the deduplication of the commitments, the groupings of the cells the device
// kernels walk, and the Fiat-Shamir challenge.  Also hash_to_bls_field, which every KZG challenge of the library ends in.
//
// Plain C++ with no CUDA types, so that tests can build it into a CPU program (tests/cell_batch_check.cpp).
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

namespace b200zk {

constexpr uint32_t kBatchBlobN = 4096;    // FIELD_ELEMENTS_PER_BLOB
constexpr uint32_t kBatchCells = 128;     // CELLS_PER_EXT_BLOB: a cell index is below it
constexpr uint32_t kBatchCellN = 64;      // FIELD_ELEMENTS_PER_CELL
constexpr size_t kBatchCellBytes = 2048;  // BYTES_PER_CELL

// the digest read as a big-endian integer and reduced mod r, the BLS12-381 group order; 32 bytes big-endian out
void hash_to_bls_field(const uint8_t digest[32], uint8_t out_be[32]);

// n cells k = 0..n-1, each with a 48-byte commitment and a cell index
struct CellBatch {
  size_t n = 0;
  // the spec's deduplicated commitments, in order of first occurrence: unique[i] is the first cell whose commitment is
  // commitment i; commit_index[k] is cell k's commitment index (commitment_indices of the spec)
  std::vector<uint32_t> unique, commit_index;
  // cells grouped by commitment: commitment i's cells are by_commit[commit_off[i] .. commit_off[i + 1]), ascending in k
  std::vector<uint32_t> commit_off, by_commit;
  // cells grouped by the cell indices that occur, ascending: columns[q] is the q-th such index, and its cells are
  // by_column[column_off[q] .. column_off[q + 1]), ascending in k
  std::vector<uint32_t> columns, column_off, by_column;
};

// The index check, then the deduplication and both groupings (counting sorts, stable in k).  Returns n when every cell
// index is below 128 and *out is filled, else the first cell whose index is not (and *out is left unspecified).
size_t cell_batch_build(const uint8_t* commitments /* 48 n */, const uint64_t* cell_indices, size_t n, CellBatch* out);

// compute_verify_cell_kzg_proof_batch_challenge: hash_to_bls_field(SHA-256("RCKZGCBATCH__V1_" | 4096, 64, the number of
// deduplicated commitments, n as u64 big-endian | the deduplicated commitments | for each cell k: its commitment index
// and cell index as u64 big-endian, its 2048 bytes, its proof)), from the caller's buffers
void cell_batch_challenge(const CellBatch& b, const uint8_t* commitments /* 48 n */, const uint64_t* cell_indices, const uint8_t* cells /* 2048 n */,
                          const uint8_t* proofs /* 48 n */, uint8_t r_be[32]);

}  // namespace b200zk
