// HNSW dense search engine on one H100.
//
// Replaces (reference, CPU/OpenMP, one Searcher per thread):
//   c_ann_hnsw_predict_* ............. pecos/core/libpecos.cpp:527-564
//   HNSW::predict_single ............. pecos/core/ann/hnsw.hpp:927-971
//   HNSW::search_level ............... pecos/core/ann/hnsw.hpp:849-924
//   Searcher / SetOfVistedNodes ...... pecos/core/ann/hnsw.hpp:341-446   (here: per-warp bitmap + heaps in HBM/shared memory)
//   FeatVecDense{IP,L2}Simd::distance  pecos/core/ann/feat_vectors.hpp:134-162 + distance_impl/x86.hpp:121-157, :256-296
#pragma once

#include <functional>
#include <memory>
#include <vector>

#include "cuda_util.h"
#include "hnsw_host.h"

namespace pb200 {

struct HnswDev {
    const float* vec;
    const uint32_t* nbr0;
    const uint32_t* l1;
    uint32_t num_node, max_level, init_node, feat_dim;
    uint32_t vstride, main_pad, tail_len, n0stride, l0_max_degree;
    uint32_t l1_node_mem, l1_level_mem, l1_max_degree;
    int metric;
    // sparse (csr) indices: row r = entries [sp_ptr[r], sp_ptr[r+1]) of sp_ent, {index, value bits}, indices ascending
    const unsigned long long* sp_ptr;
    const uint2* sp_ent;
};

struct HnswSparseQueries {  // device CSR of the query batch (sparse indices)
    const unsigned long long* ptr;
    const uint32_t* idx;
    const float* val;
    uint32_t qcap;  // query entries staged per warp in shared memory (longer rows are searched in global memory)
};

struct HnswCounters {  // algorithmic-byte counters of SURVEY.md 8(d), totals over the last search call
    unsigned long long n_dist = 0;    // distance evaluations (one base vector read each)
    unsigned long long n_expand = 0;  // level-0 expansions (one neighbour-list read each)
    unsigned long long n_hops = 0;    // upper-level neighbourhood reads
    unsigned long long n_queries = 0;
    unsigned long long n_entries = 0;  // sparse indices: stored entries of the evaluated base rows (8 bytes each)
};

// One warp's shared-memory slice may take at most this much; also the search kernels' dynamic shared-memory limit.
constexpr uint32_t kWarpSmemMax = 200u * 1024u;

// Bytes of one warp's shared-memory slice (a multiple of 16): the staged query -- dense, the query row plus `stages` bulk-copy
// ring rows and their mbarriers; sparse, qcap indices and values plus the index filter -- followed by `tail` bytes of the
// caller's own.
uint32_t warp_smem_bytes(bool sparse, uint32_t vstride, int stages, uint32_t qcap, uint32_t tail);

// CTA shape of a search launch with `per_warp` bytes of shared memory per warp: 8 warps per CTA, halved while a CTA would
// take more than 96 KB; as many CTAs per SM (at least one) as max_warps_per_sm warps and 220 KB of shared memory allow.
struct CtaShape {
    uint32_t warps, ctas_per_sm, sms;
};
CtaShape cta_shape(int device, uint32_t per_warp, uint32_t max_warps_per_sm);

// Launch plan of one search with a result heap of ef = max(efS, topk) entries: the ring depth, where the result heap lives and
// the bytes of one warp's shared-memory slice [staged query | ring rows | mbarriers | nbmax neighbour ids | distances | result
// heap if held in shared memory].  Tried in order, the first that fits kWarpSmemMax wins: the heap in shared memory (only while
// ef <= kEfSmemMax) at ring depths `stages`, 4, 0; then the heap in global memory at the same depths.  So a dense index serves
// every ef up to the width that fits with the heap in global memory at depth 0 (vstride * 4 + nbmax * 8 bytes); fits = false
// beyond it.  Sparse indices always run depth 0 and fit for every width.  Results do not depend on the plan.
constexpr uint32_t kEfSmemMax = 512;
struct HnswPlan {
    bool fits;
    int stages;
    bool heap_in_smem;
    uint32_t per_warp;
    uint32_t nbmax;  // neighbour slots of the slice: the longest neighbour list, rounded up to 32
};
HnswPlan hnsw_plan(bool sparse, uint32_t vstride, uint32_t max_degree, int stages, uint32_t ef, uint32_t qcap);

// A query batch in HBM, as the search kernels take it: dense rows, or csr rows with offsets rebased to the batch.
class DeviceQueries {
public:
    // the first `rows` rows of x, on `stream`; returns once x is no longer read
    void upload(const HostMatrix& x, uint32_t rows, cudaStream_t stream);
    const float* dense() const { return val_.get(); }  // dense rows (csr: the values)
    HnswSparseQueries sparse() const { return HnswSparseQueries{ptr_.get(), idx_.get(), val_.get(), qcap_}; }
    uint32_t qcap() const { return qcap_; }  // csr: entries staged per warp (the longest row, rounded up to 32, at most kSpQcapMax)

private:
    DeviceBuffer<float> val_;
    DeviceBuffer<unsigned long long> ptr_;
    DeviceBuffer<uint32_t> idx_;
    uint32_t qcap_ = 0;
};

// The base rows in HBM as the search kernels read them (layouts in hnsw_host.h): dense rows in the permuted layout, or
// sparse rows as sp_ptr offsets and interleaved {index, value bits} entries.
class DeviceRows {
public:
    // row(r, &val, &idx): the values of row r and, sparse, its ascending indices; returns its stored entries (dense: feat_dim)
    using RowFn = std::function<uint32_t(uint64_t r, const float** val, const uint32_t** idx)>;
    // uploads rows [0, n) on `stream`, sets the row fields of *view (vec, vstride, main_pad, tail_len, sp_ptr, sp_ent) and
    // returns the bytes placed in HBM
    uint64_t upload(uint64_t n, uint32_t feat_dim, bool sparse, const RowFn& row, cudaStream_t stream, HnswDev* view);

private:
    DeviceBuffer<float> vec_;
    DeviceBuffer<unsigned long long> sp_ptr_;
    DeviceBuffer<uint2> sp_ent_;
};

class HnswEngine {
public:
    HnswEngine(std::unique_ptr<HnswHostIndex> host, int device);
    ~HnswEngine();

    const HnswHostIndex& host() const { return *host_; }
    int metric() const { return host_->metric; }
    bool sparse() const { return host_->sparse; }

    // Host-buffer entry point: x holds nq queries, dense rows for a dense index or csr rows (column indices ascending within a
    // row) for a sparse one, whose distances are ordered sparse intersections; ret arrays nq x topk (caller-zeroed, like the
    // reference).
    void predict(const HostMatrix& x, uint32_t efS, uint32_t topk, uint32_t* ret_idx, float* ret_val);

    // Device-resident queries (bench "value" leg).
    void resident_upload(const HostMatrix& x);
    double resident_predict(uint32_t efS, uint32_t topk);  // returns device ms of the search kernel
    void resident_fetch(uint32_t* ret_idx, float* ret_val);

    // Index sharding (one graph per shard, one engine per rank).  sharded_local_packed searches this shard and writes
    // [nq][topk] 16-byte ShardRecords (shard_merge.cuh) to the caller-owned device buffer rec_dev:
    //   key = (~orderable(dist) << 32) | ~(rank * topk + slot), id = id_offset + local id, val = dist; key 0 = empty slot.
    // sharded_merge_packed merges the all-gathered [world][rows][topk] records into ret arrays rows x topk; rows with fewer
    // than topk results keep zeros, as in predict.
    void sharded_local_packed(const HostMatrix& x, uint32_t efS, uint32_t topk, uint32_t rank, uint32_t id_offset, void* rec_dev);
    void sharded_merge_packed(uint32_t world, uint32_t rows, uint32_t topk, const void* g_rec, uint32_t* ret_idx, float* ret_val);

    HnswCounters counters();
    uint64_t launches() const { return launches_; }
    uint32_t vcap_retries() const { return vcap_retries_; }  // batches re-run after a candidate-queue overflow
    uint64_t index_bytes() const { return index_bytes_; }
    double last_kernel_ms() const { return last_ms_; }
    // rows kept in flight per warp by the bulk-copy ring: 0 (direct loads), 4 or 8, used wherever the ring fits (see
    // ensure_scratch_)
    void set_stages(int stages);
    int stages() const { return stages_; }
    // the last search launch: {ring depth it ran, warps per CTA, CTAs, dynamic shared memory per CTA (bytes),
    // result-heap entries held in global scratch (0 while every heap fitted in shared memory)}
    void launch_info(uint64_t* out) const;
    // the plan a search (efS, topk) on this index will run with (sparse: for the longest query rows a batch can stage);
    // host-only, so callers can refuse a search that does not fit before making it
    HnswPlan search_plan(uint32_t efS, uint32_t topk) const;

private:
    // selects the device, checks x against the index and uploads it into `into`, unless there is nothing to search (no rows
    // or topk 0): returns whether it did
    bool upload_(const HostMatrix& x, uint32_t topk, DeviceQueries& into);
    // the launch geometry follows the staging capacity qcap of the queries searched
    void ensure_scratch_(uint32_t ef, uint32_t qcap);
    HnswPlan plan_(uint32_t ef, uint32_t qcap) const;
    struct SearchIo {  // the first nq rows of *queries, searched into idx / val ([nq][topk])
        const DeviceQueries* queries;
        uint32_t nq;
        uint32_t* idx;
        float* val;
    };
    // idx_fill: byte value io.idx is filled with before the search (0: the reference's zeros; 0xFF: empty slots read
    // 0xFFFFFFFF, which no node id can be, for the shard pack kernel)
    double launch_(const SearchIo& io, uint32_t efS, uint32_t topk, int idx_fill = 0);
    double launch_once_(const SearchIo& io, uint32_t efS, uint32_t topk, int idx_fill, bool* overflow);

    std::unique_ptr<HnswHostIndex> host_;
    int device_ = 0;
    cudaStream_t stream_ = nullptr;
    cudaEvent_t ev_[2] = {nullptr, nullptr};
    DeviceRows rows_;
    DeviceBuffer<uint32_t> nbr0_;
    DeviceBuffer<uint32_t> l1_;
    HnswDev view_{};
    uint64_t index_bytes_ = 0;

    // per-warp scratch
    uint32_t n_warps_ = 0, warps_per_cta_ = 0, n_ctas_ = 0;
    HnswPlan run_plan_{};  // plan of the current launch geometry (ensure_scratch_): its ring depth is stages_ or shallower
    uint32_t last_ctas_ = 0, last_smem_ = 0;
    uint32_t vcap_ = 0;
    uint32_t vcap_floor_ = 0;    // minimum candidate-queue capacity (doubled after an overflow)
    uint32_t vcap_retries_ = 0;
    DeviceBuffer<uint32_t> bitmap_;
    DeviceBuffer<uint32_t> vlist_;
    DeviceBuffer<uint2> cand_;
    DeviceBuffer<uint2> topk_heap_;
    DeviceBuffer<unsigned long long> ctrl_;  // [0] query counter, [1] error flag, [2..5] counters

    DeviceQueries queries_;  // host-buffer calls
    DeviceBuffer<uint32_t> out_idx_;
    DeviceBuffer<float> out_val_;
    DeviceBuffer<uint32_t> merge_cnt_;  // per-query result counts of the shard merge
    // the resident batch owns its queries and results: host-buffer calls in between change neither
    DeviceQueries res_queries_;
    DeviceBuffer<uint32_t> res_idx_;
    DeviceBuffer<float> res_val_;
    uint32_t res_nq_ = 0, res_topk_ = 0;

    uint64_t launches_ = 0;
    double last_ms_ = 0.0;
    int stages_ = 4;
};

}  // namespace pb200
