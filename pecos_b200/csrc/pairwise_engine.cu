// PairwiseANN search on H100 (sm_90a).  See pairwise_engine.h for the reference map.
//
// Column lengths are heavy-tailed, so the work is balanced by rows, not by pairs.  Two kernels per tile of pairs:
//   1. pw_distance_kernel: work items of (pair, slice of at most kSlice positions of its column), claimed from an atomic
//      counter.  A warp stages the item's query (kept while consecutive items share it, so an is_same_input batch stages it
//      once per warp), evaluates the slice's distances with the HNSW distance code (batch_distances / batch_distances_sparse,
//      the same bits as the reference's ip distances) and writes {distance bits, position} into the pair's scratch region.
//   2. pw_select_kernel: one warp per pair, k = min(topk, n).  A radix select finds the k-th smallest distance T.  When
//      the column holds no NaN distance, exactly one entry equals T and the k smallest are pairwise distinct, every heap
//      sequence ends in the same sorted list, so the k smallest sorted ascending ARE the reference's answer (fast path; with
//      a NaN, `<` is no strict weak order and the heap leaves it wherever the sequence puts it).  Otherwise one lane replays the
//      reference's push-all / pop-to-k / sort_heap over the column in stored order with the restated libstdc++ heap
//      algorithms (in shared memory when the column fits, in place in the pair's global scratch otherwise), which settles
//      every tie exactly as the CPU code does.
#include "pairwise_engine.h"
#include "hnsw_device.cuh"
#include "shard_merge.cuh"

#include <algorithm>
#include <cstring>

namespace pb200 {

namespace {

constexpr uint32_t kSlice = 128;         // column positions per distance work item
constexpr uint32_t kSelCap = 1024;       // fast path: k up to this; replay in shared memory: n up to this
constexpr int kSelectWarps = 4;          // pairs per CTA of the select kernel
constexpr uint64_t kTileEntries = 1ull << 25;  // column entries per tile (scratch: 8 bytes each)

// distances of the work items' slices -> scratch
template <int STAGES, bool SPARSE>
__global__ void __launch_bounds__(256)
pw_distance_kernel(const HnswDev ix, const float* __restrict__ Q, const HnswSparseQueries SQ, const uint4* __restrict__ pairs,
                   const unsigned long long* __restrict__ pair_off, const uint2* __restrict__ items, const uint32_t n_items,
                   const uint32_t* __restrict__ row_idx, uint2* __restrict__ scratch, const uint32_t per_warp_bytes,
                   unsigned long long* ctrl) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    unsigned char* base = smem_raw + static_cast<size_t>(warp) * per_warp_bytes;
    // per-warp slice: dense [query | STAGES ring rows | STAGES mbarriers | distances]; sparse [query indices | values | filter | distances]
    float* qs = reinterpret_cast<float*>(base);
    float* ring = qs + ix.vstride;
    unsigned long long* mbars = reinterpret_cast<unsigned long long*>(ring + static_cast<size_t>(STAGES) * ix.vstride);
    uint32_t* sq_idx = reinterpret_cast<uint32_t*>(base);
    float* sq_val = reinterpret_cast<float*>(sq_idx + SQ.qcap);
    uint32_t* sq_filter = reinterpret_cast<uint32_t*>(sq_val + SQ.qcap);
    float* dist = SPARSE ? reinterpret_cast<float*>(sq_filter + kSpFilterWords) : reinterpret_cast<float*>(mbars + STAGES);
    const uint32_t mbar0 = smem_addr(mbars);
    uint32_t phase_bits = 0;
    if (STAGES > 0 && !SPARSE) {
        if (lane == 0) {
            for (int s = 0; s < STAGES; ++s) mbar_init(mbar0 + 8u * s, 1u);
            fence_proxy_async_smem();
        }
        __syncwarp();
    }
    const uint32_t d = ix.feat_dim;
    uint32_t staged = 0xFFFFFFFFu;
    SparseQuery sq{nullptr, nullptr, 0u, sq_filter};
    unsigned long long n_entries = 0;
    for (;;) {
        unsigned long long it = 0;
        if (lane == 0) it = atomicAdd(&ctrl[0], 1ull);
        it = __shfl_sync(kFull, it, 0);
        if (it >= n_items) break;
        const uint2 item = items[it];
        const uint4 pr = pairs[item.x];
        const uint32_t q = pr.x;
        const uint32_t cnt = min(kSlice, pr.y - item.y);
        const uint64_t col0 = (static_cast<uint64_t>(pr.w) << 32) | pr.z;
        if (q != staged) {
            staged = q;
            if (SPARSE) {
                const unsigned long long q0 = SQ.ptr[q];
                sq.n = static_cast<uint32_t>(SQ.ptr[q + 1] - q0);
                for (uint32_t w = lane; w < kSpFilterWords; w += 32) sq_filter[w] = 0u;
                __syncwarp();
                const bool in_smem = sq.n <= SQ.qcap;
                for (uint32_t i = lane; i < sq.n; i += 32) {
                    const uint32_t c = SQ.idx[q0 + i];
                    if (in_smem) { sq_idx[i] = c; sq_val[i] = SQ.val[q0 + i]; }
                    const uint32_t h = sp_hash(c);
                    atomicOr(&sq_filter[h >> 5], 1u << (h & 31u));
                }
                sq.idx = in_smem ? sq_idx : SQ.idx + q0;
                sq.val = in_smem ? sq_val : SQ.val + q0;
                __syncwarp();
            } else {
                for (uint32_t i = lane; i < ix.vstride; i += 32) qs[i] = 0.0f;
                __syncwarp();
                const float* qrow = Q + static_cast<uint64_t>(q) * d;
                for (uint32_t i = lane; i < d; i += 32) qs[permuted_pos_dev(ix, i)] = qrow[i];
                __syncwarp();
            }
        }
        const uint32_t* ids = row_idx + col0 + item.y;
        if (SPARSE) batch_distances_sparse<HNSW_IP>(ix, sq, ids, dist, cnt, lane, n_entries);
        else batch_distances<HNSW_IP, STAGES>(ix, qs, ids, dist, cnt, lane, ring, mbar0, phase_bits);
        uint2* out = scratch + pair_off[item.x] + item.y;
        for (uint32_t i = lane; i < cnt; i += 32) out[i] = make_uint2(__float_as_uint(dist[i]), item.y + i);
        __syncwarp();
    }
    if (SPARSE) {
        n_entries += __shfl_xor_sync(kFull, n_entries, 16);
        if (lane == 0 && n_entries) atomicAdd(&ctrl[1], n_entries);
    }
}

// sort key of a distance: -0.0 folded onto +0.0 so that equal floats have equal keys
__device__ __forceinline__ uint32_t dist_key(uint32_t bits) { return orderable(__fadd_rn(__uint_as_float(bits), 0.0f)); }

// one warp per pair: exact top-k of the pair's scratch -> the caller's slots
__global__ void __launch_bounds__(kSelectWarps * 32)
pw_select_kernel(const uint4* __restrict__ pairs, const unsigned long long* __restrict__ pair_off, const uint32_t n_pairs,
                 const uint32_t topk, uint2* scratch, const uint32_t* __restrict__ row_idx, const float* __restrict__ y_val,
                 uint32_t* __restrict__ oI, uint32_t* __restrict__ oM, float* __restrict__ oD, float* __restrict__ oV,
                 const uint64_t out_pair0, unsigned long long* ctrl) {
    __shared__ uint32_t hist_all[kSelectWarps][256];
    __shared__ unsigned long long buf_all[kSelectWarps][kSelCap];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    uint32_t* hist = hist_all[warp];
    unsigned long long* buf = buf_all[warp];
    const uint32_t n_warps = gridDim.x * kSelectWarps;
    for (uint32_t p = blockIdx.x * kSelectWarps + warp; p < n_pairs; p += n_warps) {
        const uint4 pr = pairs[p];
        const uint32_t n = pr.y;
        if (n == 0) continue;
        const uint64_t col0 = (static_cast<uint64_t>(pr.w) << 32) | pr.z;
        const uint32_t k = min(topk, n);
        uint2* e = scratch + pair_off[p];

        // ---- radix select of the k-th smallest key T, 8 bits per pass; the first pass also looks for NaN distances
        uint32_t prefix = 0, rank = k, eq = 0;
        bool nan = false;
        for (int shift = 24; shift >= 0; shift -= 8) {
            for (int b = lane; b < 256; b += 32) hist[b] = 0u;
            __syncwarp();
            const uint32_t hmask = (shift == 24) ? 0u : (0xFFFFFFFFu << (shift + 8));
            for (uint32_t i = lane; i < n; i += 32) {
                const uint32_t bits = e[i].x;
                if (shift == 24) nan |= (bits << 1) > 0xFF000000u;  // isnan, whatever the sign and payload
                const uint32_t key = dist_key(bits);
                if ((key & hmask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
            }
            __syncwarp();
            uint32_t c[8], s = 0;
#pragma unroll
            for (int j = 0; j < 8; ++j) { c[j] = hist[8 * lane + j]; s += c[j]; }
            uint32_t incl = s;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t v = __shfl_up_sync(kFull, incl, o);
                if (lane >= o) incl += v;
            }
            const int owner = __ffs(__ballot_sync(kFull, incl >= rank)) - 1;
            uint32_t bin = 0, below = 0, cnt = 0;
            if (lane == owner) {
                uint32_t run = incl - s;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    if (cnt == 0 && run + c[j] >= rank) { bin = 8 * lane + j; below = run; cnt = c[j]; }
                    run += c[j];
                }
            }
            bin = __shfl_sync(kFull, bin, owner);
            below = __shfl_sync(kFull, below, owner);
            eq = __shfl_sync(kFull, cnt, owner);
            prefix |= bin << shift;
            rank -= below;
            __syncwarp();
        }
        const uint32_t T = prefix;

        // ---- fast path: no NaN in the column, the k entries with key <= T sorted by (key, position), all keys distinct
        bool fast = (eq == 1u) && (k <= kSelCap) && !__any_sync(kFull, nan);
        if (fast) {
            uint32_t got = 0;
            for (uint32_t b0 = 0; b0 < n; b0 += 32) {
                const uint32_t i = b0 + lane;
                uint32_t key = 0;
                const bool take = i < n && (key = dist_key(e[i].x)) <= T;
                const unsigned m = __ballot_sync(kFull, take);
                if (take) buf[got + __popc(m & ((1u << lane) - 1u))] = (static_cast<unsigned long long>(key) << 32) | i;
                got += __popc(m);
            }
            uint32_t P = 1;
            while (P < k) P <<= 1;
            for (uint32_t i = k + lane; i < P; i += 32) buf[i] = ~0ull;
            __syncwarp();
            for (uint32_t size = 2; size <= P; size <<= 1) {
                for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
                    for (uint32_t i = lane; i < P; i += 32) {
                        const uint32_t j = i ^ stride;
                        if (j > i) {
                            const unsigned long long a = buf[i], b = buf[j];
                            if ((a > b) == ((i & size) == 0)) { buf[i] = b; buf[j] = a; }
                        }
                    }
                    __syncwarp();
                }
            }
            bool dup = false;
            for (uint32_t i = lane + 1; i < k; i += 32) dup |= (buf[i] >> 32) == (buf[i - 1] >> 32);
            fast = __ballot_sync(kFull, dup) == 0u;
            if (fast) {
                for (uint32_t j = lane; j < k; j += 32) {
                    const uint32_t pos = static_cast<uint32_t>(buf[j]);
                    const uint64_t o = (out_pair0 + p) * topk + j;
                    oI[o] = row_idx[col0 + pos];
                    oD[o] = __uint_as_float(e[pos].x);
                    oV[o] = y_val[col0 + pos];
                    oM[o] = 1u;
                }
            }
            __syncwarp();
        }
        if (fast) continue;

        // ---- replay of predict_single's heap sequence (pairwise.hpp:275-286): max-heap on distance, payload = position
        uint2* h = e;
        if (n <= kSelCap) {
            h = reinterpret_cast<uint2*>(buf);
            for (uint32_t i = lane; i < n; i += 32) h[i] = e[i];
        }
        __syncwarp();
        if (lane == 0) {
            for (uint32_t i = 1; i < n; ++i) heap_sift_up<true>(h, static_cast<int>(i), 0, h[i]);  // push_heap of every entry
            int m = static_cast<int>(n);
            while (m > static_cast<int>(k)) heap_pop<true>(h, m);
            while (m > 1) {  // std::sort_heap
                const uint2 value = h[m - 1];
                h[m - 1] = h[0];
                heap_adjust<true>(h, 0, m - 1, value);
                --m;
            }
            atomicAdd(&ctrl[2], 1ull);
        }
        __syncwarp();
        for (uint32_t j = lane; j < k; j += 32) {
            const uint2 v = h[j];
            const uint64_t o = (out_pair0 + p) * topk + j;
            oI[o] = row_idx[col0 + v.y];
            oD[o] = __uint_as_float(v.x);
            oV[o] = y_val[col0 + v.y];
            oM[o] = 1u;
        }
        __syncwarp();
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------------
PairwisePlan pairwise_plan(bool sparse, uint32_t vstride, uint32_t qcap) {
    auto per_warp_bytes = [&](int stages) { return warp_smem_bytes(sparse, vstride, stages, qcap, kSlice * 4u); };
    const int stages = (!sparse && vstride > 0 && per_warp_bytes(4) <= kWarpSmemMax) ? 4 : 0;
    const uint32_t per_warp = per_warp_bytes(stages);
    return PairwisePlan{per_warp <= kWarpSmemMax, stages, per_warp};
}

const HnswDev& PairwiseModel::device_view(int device) {
    std::lock_guard<std::mutex> lock(mu_);
    if (uploaded_) {
        if (device != device_) throw std::runtime_error("pecos_b200: a PairwiseANN model serves the device it was first searched on");
        return view_;
    }
    PB200_CUDA(cudaSetDevice(device));
    const PairwiseHostModel& H = *host_;
    cudaStream_t st = nullptr;
    PB200_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    HnswDev v{};
    v.feat_dim = H.feat_dim;
    v.metric = HNSW_IP;
    v.num_node = H.num_input_keys;
    rows_.upload(H.num_input_keys, H.feat_dim, H.sparse, [&H](uint64_t r, const float** val, const uint32_t** idx) {
        if (!H.sparse) {
            *val = H.x_val + r * H.feat_dim;
            return H.feat_dim;
        }
        *val = H.x_val + H.x_ptr[r];
        *idx = H.x_idx + H.x_ptr[r];
        return static_cast<uint32_t>(H.x_ptr[r + 1] - H.x_ptr[r]);
    }, st, &v);
    std::vector<unsigned long long> cp(H.col_ptr, H.col_ptr + static_cast<uint64_t>(H.num_label_keys) + 1);
    col_ptr_.upload(cp.data(), cp.size(), st);
    row_idx_.reserve(std::max<uint64_t>(H.nnz_y, 1));
    y_val_.reserve(std::max<uint64_t>(H.nnz_y, 1));
    if (H.nnz_y) {
        PB200_CUDA(cudaMemcpyAsync(row_idx_.get(), H.row_idx, H.nnz_y * 4, cudaMemcpyHostToDevice, st));
        PB200_CUDA(cudaMemcpyAsync(y_val_.get(), H.y_val, H.nnz_y * 4, cudaMemcpyHostToDevice, st));
    }
    PB200_CUDA(cudaStreamSynchronize(st));
    PB200_CUDA(cudaStreamDestroy(st));
    view_ = v;
    device_ = device;
    uploaded_ = true;
    return view_;
}

PairwiseSearcher::PairwiseSearcher(PairwiseModel* model, int device) : model_(model), device_(device) {
    PB200_CUDA(cudaSetDevice(device_));
    PB200_CUDA(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    for (auto& e : ev_) PB200_CUDA(cudaEventCreate(&e));
    ctrl_.reserve(4);
    PB200_CUDA(cudaMemsetAsync(ctrl_.get(), 0, 4 * sizeof(unsigned long long), stream_));
    PB200_CUDA(cudaStreamSynchronize(stream_));
}

PairwiseSearcher::~PairwiseSearcher() {
    cudaSetDevice(device_);
    if (stream_) cudaStreamSynchronize(stream_);
    for (auto& e : ev_) if (e) cudaEventDestroy(e);
    if (stream_) cudaStreamDestroy(stream_);
}

void PairwiseSearcher::predict(uint32_t batch, uint32_t topk, const HostMatrix& q, const uint32_t* label_keys, uint32_t* ret_I,
                               uint32_t* ret_M, float* ret_D, float* ret_V, bool is_same_input) {
    const PairwiseHostModel& H = model_->host();
    counters_ = PairwiseCounters{};
    last_ms_ = 0.0;
    std::fill(last_launch_, last_launch_ + 4, 0ull);
    if (batch == 0 || topk == 0) return;  // the reference writes nothing
    // every check before any GPU work: a bad label key would read out of bounds in the reference
    for (uint32_t b = 0; b < batch; ++b)
        if (label_keys[b] >= H.num_label_keys)
            throw std::runtime_error("pecos_b200: label_keys[" + std::to_string(b) + "] = " + std::to_string(label_keys[b]) +
                                     " is out of range (num_label_keys = " + std::to_string(H.num_label_keys) + ")");
    const uint32_t need_rows = is_same_input ? 1u : batch;
    if (q.rows < need_rows) throw std::runtime_error("pecos_b200: PairwiseANN query matrix has fewer rows than the batch needs");
    if (q.cols != H.feat_dim) throw std::runtime_error("pecos_b200: PairwiseANN query dimension != feat_dim");
    if ((q.row_ptr != nullptr) != H.sparse) throw std::runtime_error("pecos_b200: PairwiseANN query type differs from the model's");
    if (!H.sparse && !pairwise_plan(false, dense_vstride(H.feat_dim), 0).fits)
        throw std::runtime_error("pecos_b200: PairwiseANN feat_dim " + std::to_string(H.feat_dim) + " too large for the shared-memory "
                                 "staging area (dense models serve every d up to 51,024 and multiples of 16 up to 51,072)");

    PB200_CUDA(cudaSetDevice(device_));
    const HnswDev ix = model_->device_view(device_);

    queries_.upload(q, need_rows, stream_);  // the rows the batch uses
    const HnswSparseQueries sq = queries_.sparse();
    // the caller's result slots travel both ways: slots the reference leaves untouched stay as the caller had them
    const uint64_t n_out = static_cast<uint64_t>(batch) * topk;
    out_I_.upload(ret_I, n_out, stream_);
    out_M_.upload(ret_M, n_out, stream_);
    out_D_.upload(ret_D, n_out, stream_);
    out_V_.upload(ret_V, n_out, stream_);
    PB200_CUDA(cudaMemsetAsync(ctrl_.get(), 0, 4 * sizeof(unsigned long long), stream_));

    // launch geometry of the distance kernel (pairwise_plan): dense rows through a ring of 4 where it fits, else direct loads
    const PairwisePlan plan = pairwise_plan(H.sparse, ix.vstride, sq.qcap);
    if (!plan.fits) throw std::runtime_error("pecos_b200: PairwiseANN query too large for the shared-memory staging area");
    const int stages = plan.stages;
    const uint32_t per_warp = plan.per_warp;
    const CtaShape shape = cta_shape(device_, per_warp, 64u);
    const uint32_t warps = shape.warps, sms = shape.sms, ctas_per_sm = shape.ctas_per_sm;
    const uint32_t cta_smem = warps * per_warp;
    auto dist_kernel = H.sparse ? pw_distance_kernel<0, true> : (stages ? pw_distance_kernel<4, false> : pw_distance_kernel<0, false>);
    PB200_CUDA(cudaFuncSetAttribute(dist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(cta_smem)));

    float total_ms = 0.f;
    std::vector<uint4> pairs;
    std::vector<unsigned long long> offs;
    std::vector<uint2> items;
    for (uint32_t p0 = 0; p0 < batch;) {
        // a tile: consecutive pairs whose columns hold at most kTileEntries entries together (or one longer column)
        pairs.clear(); offs.clear(); items.clear();
        uint64_t total = 0;
        uint32_t p1 = p0;
        for (; p1 < batch; ++p1) {
            const uint32_t l = label_keys[p1];
            const uint32_t n = H.col_len(l);
            if (p1 > p0 && total + n > kTileEntries) break;
            const uint64_t c0 = H.col_ptr[l];
            const uint32_t pi = p1 - p0;
            pairs.push_back(make_uint4(is_same_input ? 0u : p1, n, static_cast<uint32_t>(c0), static_cast<uint32_t>(c0 >> 32)));
            offs.push_back(total);
            for (uint32_t s = 0; s < n; s += kSlice) items.push_back(make_uint2(pi, s));
            total += n;
        }
        const uint32_t np = p1 - p0;
        counters_.n_dist += total;
        ++last_launch_[3];
        if (total) {
            pairs_.upload(pairs.data(), np, stream_);
            pair_off_.upload(offs.data(), np, stream_);
            items_.upload(items.data(), items.size(), stream_);
            scratch_.reserve(total);
            PB200_CUDA(cudaMemsetAsync(ctrl_.get(), 0, sizeof(unsigned long long), stream_));
            const uint32_t n_items = static_cast<uint32_t>(items.size());
            const uint32_t ctas = std::max<uint32_t>(1, std::min<uint32_t>(sms * ctas_per_sm, (n_items + warps - 1) / warps));
            const uint32_t sel_ctas = std::max<uint32_t>(1, std::min<uint32_t>(sms * 16u, (np + kSelectWarps - 1) / kSelectWarps));
            PB200_CUDA(cudaEventRecord(ev_[0], stream_));
            dist_kernel<<<ctas, warps * 32, cta_smem, stream_>>>(ix, queries_.dense(), sq, pairs_.get(), pair_off_.get(), items_.get(), n_items,
                                                                model_->row_idx(), scratch_.get(), per_warp, ctrl_.get());
            PB200_CUDA(cudaGetLastError());
            pw_select_kernel<<<sel_ctas, kSelectWarps * 32, 0, stream_>>>(pairs_.get(), pair_off_.get(), np, topk, scratch_.get(),
                                                                          model_->row_idx(), model_->y_val(), out_I_.get(), out_M_.get(),
                                                                          out_D_.get(), out_V_.get(), p0, ctrl_.get());
            PB200_CUDA(cudaGetLastError());
            PB200_CUDA(cudaEventRecord(ev_[1], stream_));
            PB200_CUDA(cudaEventSynchronize(ev_[1]));  // the host vectors of this tile are reused by the next one
            float ms = 0.f;
            PB200_CUDA(cudaEventElapsedTime(&ms, ev_[0], ev_[1]));
            total_ms += ms;
        }
        p0 = p1;
    }
    PB200_CUDA(cudaMemcpyAsync(ret_I, out_I_.get(), n_out * 4, cudaMemcpyDeviceToHost, stream_));
    PB200_CUDA(cudaMemcpyAsync(ret_M, out_M_.get(), n_out * 4, cudaMemcpyDeviceToHost, stream_));
    PB200_CUDA(cudaMemcpyAsync(ret_D, out_D_.get(), n_out * 4, cudaMemcpyDeviceToHost, stream_));
    PB200_CUDA(cudaMemcpyAsync(ret_V, out_V_.get(), n_out * 4, cudaMemcpyDeviceToHost, stream_));
    unsigned long long h[4];
    PB200_CUDA(cudaMemcpyAsync(h, ctrl_.get(), sizeof(h), cudaMemcpyDeviceToHost, stream_));
    PB200_CUDA(cudaStreamSynchronize(stream_));
    counters_.pairs = batch;
    counters_.n_entries = h[1];
    counters_.replays = h[2];
    last_ms_ = total_ms;
    last_launch_[0] = static_cast<uint64_t>(stages);
    last_launch_[1] = warps;
    last_launch_[2] = per_warp;
}

void PairwiseSearcher::launch_info(uint64_t* out) const { std::copy(last_launch_, last_launch_ + 4, out); }

}  // namespace pb200
