// Finalisation of the reference's sparse (csr) distances, shared by the sparse search kernel and the sparse index builder.
#pragma once

#include "hnsw_host.h"

namespace pb200 {

// FeatVecSparse{IP,L2}Simd::distance (feat_vectors.hpp:186-210) from the ordered sum of the matched products:
// ip: 1.0 - dot ; l2: x_sq + y_sq - 2.0 * dot with x_sq = y_sq = 0 (the reference takes the squared norms as the distance of a
// row to itself), i.e. -2<x,y>.  Both evaluated in double and narrowed to float, as the reference does.
template <int METRIC>
__device__ __forceinline__ float sparse_finalize(float dot) {
    return (METRIC == HNSW_IP) ? static_cast<float>(1.0 - static_cast<double>(dot))
                               : static_cast<float>(static_cast<double>(0.0f) - 2.0 * static_cast<double>(dot));
}

}  // namespace pb200
