// Distance kernels of the sparse (csr) HNSW index builder on H100 (sm_90a).  The graph logic (levels, prefix kNN, the
// reference's selection heuristic, reverse links) is pecos_b200/hnsw_build.py, shared with the dense builder; these kernels
// replace its two distance computations for csr rows.
//
// Exactness: the reference's sparse distance (do_dot_product_sparse_block<4>, distance_impl/common.hpp:15-86, finalised by
// FeatVecSparse{IP,L2}Simd::distance, feat_vectors.hpp:186-210) adds the products of the matched entries in ascending feature
// index, starting from 0.0f, un-fused.  Both kernels produce exactly that sum for every pair, so a built graph ranks neighbours
// by the very distances the search and the reference's own train use.
//
// Block kernel (prefix kNN, q x c distance blocks): inverted index of the candidate set, one CTA per query row.  The CTA walks
// the query's features in ascending order; for each feature its threads take distinct postings of the candidate range and add
// q_f * v into the candidates' accumulators (shared memory, or the output row itself when the range does not fit), with a
// barrier between features.  Every accumulator therefore receives its matched products in ascending feature order, and only
// matched ones.  Work: sum over query entries of the postings of that feature in the range, ~ sum_f df(f)^2 over a level,
// instead of the |q| + |c| per pair of a merge.
//
// Candidate-set kernel (heuristic, C x C per node): one CTA per node, one thread per unordered pair, a sorted merge of the two
// rows straight from HBM / L2.  No staging, so rows of any length and any feature dimension work with no scratch.
#include "hnsw_build_sparse.h"

#include <cmath>

#include "cuda_util.h"
#include "sparse_distance.cuh"

namespace pb200 {

namespace {

constexpr int kThreads = 256;
constexpr uint32_t kCandMax = 512;          // widest candidate set (the reverse-link pool of the builder)
constexpr uint32_t kAccSmemMax = 96 << 10;  // accumulators up to this size live in shared memory (two CTAs per SM)

struct DeviceScope {  // selects `device` for the call, restores the caller's current device
    int prev = -1;
    explicit DeviceScope(int device) {
        PB200_CUDA(cudaGetDevice(&prev));
        if (prev != device) PB200_CUDA(cudaSetDevice(device));
    }
    ~DeviceScope() {
        int cur = -1;
        if (cudaGetDevice(&cur) == cudaSuccess && cur != prev) cudaSetDevice(prev);
    }
};

// first p in [a, b) with post[p].x >= key
__device__ __forceinline__ uint64_t lower_pos(const uint2* __restrict__ post, uint64_t a, uint64_t b, uint32_t key) {
    while (a < b) {
        const uint64_t m = a + ((b - a) >> 1);
        if (__ldg(&post[m].x) < key) a = m + 1; else b = m;
    }
    return a;
}

template <int METRIC>
__global__ void __launch_bounds__(kThreads) sparse_block_kernel(const uint64_t* __restrict__ row_ptr, const uint2* __restrict__ ent,
                                                                 const int64_t* __restrict__ q_ids, const uint64_t* __restrict__ col_ptr,
                                                                 const uint2* __restrict__ post, uint32_t c0, uint32_t nc,
                                                                 float* __restrict__ out, int acc_in_smem,
                                                                 unsigned long long* work) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint64_t* s_lo = reinterpret_cast<uint64_t*>(smem_raw);
    uint64_t* s_hi = s_lo + kThreads;
    float* s_qv = reinterpret_cast<float*>(s_hi + kThreads);
    float* out_row = out + static_cast<size_t>(blockIdx.x) * nc;
    float* acc = acc_in_smem ? (s_qv + kThreads) : out_row;
    const int tid = threadIdx.x;
    const uint32_t c1 = c0 + nc;

    for (uint32_t j = tid; j < nc; j += kThreads) acc[j] = 0.0f;
    const int64_t q = q_ids[blockIdx.x];
    const uint64_t r0 = row_ptr[q], r1 = row_ptr[q + 1];
    unsigned long long walked = 0;
    for (uint64_t f0 = r0; f0 < r1; f0 += kThreads) {
        const uint32_t nf = static_cast<uint32_t>(min(static_cast<uint64_t>(kThreads), r1 - f0));
        __syncthreads();  // the previous chunk's ranges are consumed (and the zeroed accumulators are visible)
        if (tid < nf) {
            const uint2 e = ent[f0 + tid];
            const uint64_t a = col_ptr[e.x], b = col_ptr[e.x + 1];
            const uint64_t lo = lower_pos(post, a, b, c0);
            const uint64_t hi = lower_pos(post, lo, b, c1);
            s_lo[tid] = lo;
            s_hi[tid] = hi;
            s_qv[tid] = __uint_as_float(e.y);
            walked += hi - lo;
        }
        __syncthreads();
        for (uint32_t k = 0; k < nf; ++k) {  // features in ascending index order
            const uint64_t lo = s_lo[k], hi = s_hi[k];
            const float qv = s_qv[k];
            for (uint64_t p = lo + tid; p < hi; p += kThreads) {  // distinct postings = distinct candidates: no conflicts
                const uint2 pe = __ldg(&post[p]);
                float* a = acc + (pe.x - c0);
                *a = __fadd_rn(*a, __fmul_rn(qv, __uint_as_float(pe.y)));
            }
            if (hi > lo) __syncthreads();  // uniform: every thread read the same range
        }
    }
    __syncthreads();
    for (uint32_t j = tid; j < nc; j += kThreads) out_row[j] = sparse_finalize<METRIC>(acc[j]);
    if (work && walked) atomicAdd(work, walked);
}

// ordered sum of the matched products of two rows with strictly ascending indices (a sorted merge)
__device__ __forceinline__ float sparse_dot_merge(const uint2* __restrict__ a, uint32_t na, const uint2* __restrict__ b, uint32_t nb,
                                                  uint32_t& steps) {
    float dot = 0.0f;
    if (na == 0 || nb == 0) return dot;
    uint32_t i = 0, j = 0;
    uint2 x = __ldg(a), y = __ldg(b);
    for (;;) {
        if (x.x < y.x) {
            if (++i == na) break;
            x = __ldg(a + i);
        } else if (y.x < x.x) {
            if (++j == nb) break;
            y = __ldg(b + j);
        } else {
            dot = __fadd_rn(dot, __fmul_rn(__uint_as_float(x.y), __uint_as_float(y.y)));
            if (++i == na || ++j == nb) break;
            x = __ldg(a + i);
            y = __ldg(b + j);
        }
    }
    steps += i + j;
    return dot;
}

template <int METRIC>
__global__ void __launch_bounds__(kThreads) sparse_candidate_kernel(const uint64_t* __restrict__ row_ptr, const uint2* __restrict__ ent,
                                                                     const int64_t* __restrict__ cand, uint32_t C,
                                                                     float* __restrict__ out, unsigned long long* work) {
    __shared__ uint64_t s_r0[kCandMax];
    __shared__ uint32_t s_len[kCandMax];
    __shared__ int s_valid[kCandMax];
    const int64_t* c = cand + static_cast<size_t>(blockIdx.x) * C;
    float* o = out + static_cast<size_t>(blockIdx.x) * C * C;
    for (uint32_t i = threadIdx.x; i < C; i += kThreads) {
        const int64_t r = c[i];
        s_valid[i] = r >= 0;
        s_r0[i] = r >= 0 ? row_ptr[r] : 0;
        s_len[i] = r >= 0 ? static_cast<uint32_t>(row_ptr[r + 1] - row_ptr[r]) : 0;
    }
    __syncthreads();
    uint32_t steps = 0;
    for (uint32_t t = threadIdx.x; t < C * C; t += kThreads) {
        const uint32_t i = t / C, j = t - i * C;
        if (j < i) continue;  // the lower triangle is written with its mirror (the sum is symmetric bit for bit)
        float d = INFINITY;
        if (s_valid[i] && s_valid[j]) d = sparse_finalize<METRIC>(sparse_dot_merge(ent + s_r0[i], s_len[i], ent + s_r0[j], s_len[j], steps));
        o[static_cast<size_t>(i) * C + j] = d;
        o[static_cast<size_t>(j) * C + i] = d;
    }
    if (work) {
        const unsigned total = __reduce_add_sync(0xFFFFFFFFu, steps);
        if ((threadIdx.x & 31) == 0 && total) atomicAdd(work, static_cast<unsigned long long>(total));
    }
}

void check_launch(const char* what) {
    const cudaError_t err = cudaGetLastError();
    if (err != cudaSuccess) cuda_check(err, what, __FILE__, __LINE__);
}

}  // namespace

void sparse_block_distances(int device, int metric, const uint64_t* row_ptr, const uint2* ent, const int64_t* q_ids, uint32_t nq,
                            const uint64_t* col_ptr, const uint2* post, uint32_t c0, uint32_t nc, float* out,
                            unsigned long long* work, cudaStream_t stream) {
    if (metric != HNSW_IP && metric != HNSW_L2) throw std::invalid_argument("sparse_block_distances: metric must be 0 (ip) or 1 (l2)");
    if (nq == 0 || nc == 0) return;
    DeviceScope scope(device);
    const size_t head = kThreads * (2 * sizeof(uint64_t) + sizeof(float));
    const size_t acc = static_cast<size_t>(nc) * sizeof(float);
    const int in_smem = acc <= kAccSmemMax;
    const size_t smem = head + (in_smem ? acc : 0);
    auto kernel = metric == HNSW_IP ? sparse_block_kernel<HNSW_IP> : sparse_block_kernel<HNSW_L2>;
    PB200_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(head + kAccSmemMax)));
    kernel<<<nq, kThreads, smem, stream>>>(row_ptr, ent, q_ids, col_ptr, post, c0, nc, out, in_smem, work);
    check_launch("sparse_block_kernel launch");
}

void sparse_candidate_distances(int device, int metric, const uint64_t* row_ptr, const uint2* ent, const int64_t* cand, uint32_t n,
                                uint32_t C, float* out, unsigned long long* work, cudaStream_t stream) {
    if (metric != HNSW_IP && metric != HNSW_L2)
        throw std::invalid_argument("sparse_candidate_distances: metric must be 0 (ip) or 1 (l2)");
    if (C > kCandMax) throw std::invalid_argument("sparse_candidate_distances: candidate sets are limited to 512 slots");
    if (n == 0 || C == 0) return;
    DeviceScope scope(device);
    auto kernel = metric == HNSW_IP ? sparse_candidate_kernel<HNSW_IP> : sparse_candidate_kernel<HNSW_L2>;
    kernel<<<n, kThreads, 0, stream>>>(row_ptr, ent, cand, C, out, work);
    check_launch("sparse_candidate_kernel launch");
}

}  // namespace pb200
