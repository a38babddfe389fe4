// Sparse x sparse matrix product on one H100, bit-identical to the reference's smat_x_smat.
//
// Replaces (reference, CPU/OpenMP, one output row per thread):
//   c_sparse_matmul_{csr,csc}_f32 ... pecos/core/libpecos.cpp:320-335
//   smat_x_smat ..................... pecos/core/utils/matrix.hpp:1062-1290
//
// Both entry points reduce to "A x B, row by row of A" (csr: A = X, B = Y; csc: A = Y's columns, B = X's columns).  Output
// row i gets, for each A entry s in stored order and then each entry t of B row A.idx[s] in stored order, acc = acc + a_s*b_t
// (separate roundings, acc starting at +0.0f) per output index; its indices come ascending (sorted) or in first-touch order.
#pragma once

#include <cstdint>

#include "../../include/pecos_b200.h"

namespace pb200 {

// A compressed operand: `rows` rows of u64 pointers / u32 indices / f32 values (a csr matrix, or a csc matrix's columns).
struct SpmmOperand {
    uint32_t rows;
    const uint64_t* ptr;
    const uint32_t* idx;
    const float* val;
};

// Tier thresholds (DESIGN §4.9).  Symbolic pass: rows with at most kCountWarpMaxProducts products count their distinct
// outputs in one warp with a shared-memory hash set, longer rows in one CTA with a global bitmap of the output width.
// Numeric pass: rows with at most kFoldWarpMaxDistinct distinct outputs and kFoldWarpMaxProducts products fold in one warp
// with a shared-memory hash accumulator, the others in one CTA with a global-memory accumulator of 2-4x their distinct outputs.
constexpr uint64_t kCountWarpMaxProducts = 1024;
constexpr uint32_t kFoldWarpMaxDistinct = 512;
constexpr uint64_t kFoldWarpMaxProducts = 65536;

// last_info layout: {A rows, products, allocator nnz, nnz kept, count-warp rows, count-CTA rows, fold-warp rows,
// fold-CTA rows, tiles, launches}
constexpr int kSpmmInfoLen = 10;

// Computes A x B (B rows of width `width`) on `device` and hands the result to pred_alloc(col_major, alloc_rows, alloc_cols,
// nnz) once, from the calling thread.  Validates shapes and indices first (throws before any launch).  Calls on one device
// are serialised.  info (kSpmmInfoLen) and kernel_ms describe the call.
void spmm_run(int device, const SpmmOperand& A, const SpmmOperand& B, uint32_t width, bool col_major, uint64_t alloc_rows,
              uint64_t alloc_cols, py_sparse_allocator_t pred_alloc, bool eliminate_zeros, bool sorted_indices,
              uint64_t* info, double* kernel_ms);

// Device bytes a product with this B needs at least (B arrays, its row flags and the minimum workspace).
uint64_t spmm_min_bytes(uint32_t b_rows, uint64_t b_nnz);

}  // namespace pb200
