// Distance kernels of the sparse (csr) HNSW index builder (pecos_b200/hnsw_build.py); C ABI in c_api.cu.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

namespace pb200 {

// Base rows: row r = entries [row_ptr[r], row_ptr[r+1]) of ent, {u32 index, f32 value bits}, indices strictly ascending.
// Candidate set of the block kernel: its inverted index, column f = postings [col_ptr[f], col_ptr[f+1]) of post,
// {u32 position in the candidate set, f32 value bits}, positions ascending within a column.
// Every distance is bit-identical to the reference's FeatVecSparse{IP,L2}Simd::distance of the two rows.
// work (may be null): += postings walked (block) / row entries walked by the intersections (candidate sets).

// out[q * nc + (p - c0)] = distance(row q_ids[q], candidate at position p) for p in [c0, c0 + nc)
void sparse_block_distances(int device, int metric, const uint64_t* row_ptr, const uint2* ent, const int64_t* q_ids, uint32_t nq,
                            const uint64_t* col_ptr, const uint2* post, uint32_t c0, uint32_t nc, float* out,
                            unsigned long long* work, cudaStream_t stream);

// cand [n, C] row ids (-1 = empty slot); out[t, i, j] = distance(cand[t, i], cand[t, j]), +inf where a slot is empty
void sparse_candidate_distances(int device, int metric, const uint64_t* row_ptr, const uint2* ent, const int64_t* cand, uint32_t n,
                                uint32_t C, float* out, unsigned long long* work, cudaStream_t stream);

}  // namespace pb200
