// PairwiseANN search on one H100: for each (query, label) pair, the only_topk rows of column `label` of Y_csc nearest to the
// query, exactly as the reference's brute force returns them.
//
// Replaces (reference, CPU/OpenMP, one Searcher per thread):
//   c_pairwise_ann_predict_* ........ pecos/core/libpecos.cpp:628-657
//   PairwiseANN::predict_single ..... pecos/core/ann/pairwise.hpp:265-288   (push every column entry into a max-heap in stored
//                                                                           order, pop down to topk, sort_heap)
//   FeatVecDenseIPSimd / FeatVecSparseIPSimd::distance (the same distance code as the HNSW ip search)
#pragma once

#include <memory>
#include <mutex>
#include <vector>

#include "cuda_util.h"
#include "hnsw_engine.h"
#include "pairwise_host.h"

namespace pb200 {

// The model: host arrays (kept for save) plus, from the first search on, their device copies, shared read-only by every
// searcher of the model.
class PairwiseModel {
public:
    explicit PairwiseModel(std::unique_ptr<PairwiseHostModel> host) : host_(std::move(host)) {}
    const PairwiseHostModel& host() const { return *host_; }
    // uploads the arrays to `device` on first use (thread-safe); returns the device view
    const HnswDev& device_view(int device);
    const unsigned long long* col_ptr() const { return col_ptr_.get(); }
    const uint32_t* row_idx() const { return row_idx_.get(); }
    const float* y_val() const { return y_val_.get(); }
    int device() const { return device_; }

private:
    std::unique_ptr<PairwiseHostModel> host_;
    std::mutex mu_;
    bool uploaded_ = false;
    int device_ = 0;
    HnswDev view_{};
    DeviceRows rows_;  // X_trn, as the HNSW distance code reads it
    DeviceBuffer<unsigned long long> col_ptr_;
    DeviceBuffer<uint32_t> row_idx_;
    DeviceBuffer<float> y_val_;
};

// The distance kernel's per-warp shared-memory slice: [staged query | ring rows | distances of a 128-row slice].  Dense rows
// go through a bulk-copy ring of 4 rows where the slice then fits kWarpSmemMax, else they are loaded directly; a dense model
// whose row stride (dense_vstride) overflows the slice even then cannot be searched: every d up to 51,024 and every multiple of
// 16 up to 51,072 fits, nothing else does.  Host arithmetic only; the engine launches with exactly this plan.
struct PairwisePlan {
    bool fits;
    int stages;         // ring depth: 4, or 0 (direct loads)
    uint32_t per_warp;  // bytes of one warp's slice at that depth
};
PairwisePlan pairwise_plan(bool sparse, uint32_t vstride, uint32_t qcap);

struct PairwiseCounters {  // totals over the searcher's last predict call
    unsigned long long pairs = 0;
    unsigned long long n_dist = 0;     // distances evaluated (sum of the pairs' column lengths)
    unsigned long long n_entries = 0;  // sparse: stored entries of the rows read
    unsigned long long replays = 0;    // pairs whose selection was replayed with the reference's heap sequence
};

// One searcher token: its own stream and scratch.  Calls on one searcher are serialised by the caller (c_api.cu).
class PairwiseSearcher {
public:
    PairwiseSearcher(PairwiseModel* model, int device);
    ~PairwiseSearcher();
    // Host buffers in and out.  q: dense or csr query rows, of the model's kind.
    // ret_* hold batch x topk slots; only slot k < min(topk, column length) of each pair is written.
    void predict(uint32_t batch, uint32_t topk, const HostMatrix& q, const uint32_t* label_keys, uint32_t* ret_I, uint32_t* ret_M,
                 float* ret_D, float* ret_V, bool is_same_input);
    PairwiseCounters counters() const { return counters_; }
    double last_kernel_ms() const { return last_ms_; }
    // the last predict call: {ring depth of the distance kernel, warps per CTA, per-warp shared-memory bytes, tiles}; all 0
    // when it had nothing to search (batch or topk 0)
    void launch_info(uint64_t* out) const;

private:
    PairwiseModel* model_;
    int device_ = 0;
    cudaStream_t stream_ = nullptr;
    cudaEvent_t ev_[2] = {nullptr, nullptr};
    DeviceQueries queries_;
    DeviceBuffer<uint4> pairs_;    // per pair: {query row, column length, column start (u64 as 2 words)}
    DeviceBuffer<unsigned long long> pair_off_;  // per pair: offset of its scratch
    DeviceBuffer<uint2> items_;    // distance work items {pair, first position}
    DeviceBuffer<uint2> scratch_;  // {distance bits, position in the column} per column entry of the tile's pairs
    DeviceBuffer<uint32_t> out_I_, out_M_;
    DeviceBuffer<float> out_D_, out_V_;
    DeviceBuffer<unsigned long long> ctrl_;  // [0] item counter, [1] sparse entries, [2] replays
    PairwiseCounters counters_;
    double last_ms_ = 0.0;
    uint64_t last_launch_[4] = {0, 0, 0, 0};
};

}  // namespace pb200
