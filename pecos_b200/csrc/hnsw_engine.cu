// HNSW dense search on H100 (sm_90a): one warp walks one query (see hnsw_engine.h for the reference map).
//
// Per expansion of the best-first search the warp
//   A. reads the node's neighbour list, test-and-sets the per-warp visited bitmap, compacts the not-yet-visited ids in
//      list order (ballot + popc),
//   B. evaluates ALL their distances, two at a time (one per half-warp).  A half-warp's 16 lanes read one float4 each
//      per 64 components from the permuted row (256 contiguous bytes) and lane j runs exactly the accumulation chain of
//      SIMD lane j of the reference's avx512 kernel: un-fused multiply/add, fold 16 -> 4 -> 1 in the same association,
//      4-wide tail un-fused, scalar tail fused (as GCC compiles that clone) -- distances are bit-identical,
//   C. lane 0 replays the reference's queue updates sequentially in neighbour order with restated libstdc++
//      push_heap / pop_heap, so ties and the evolving upper bound behave exactly like the CPU code.
// The reference evaluates the distance of every unvisited neighbour before touching the queues (hnsw.hpp:897-914), which
// is what makes step B independent of step C.
//
// Sparse (csr) indices (FeatVecSparse{IP,L2}Simd, feat_vectors.hpp:186-210) use the same walk; only step B differs: a half-warp
// streams the neighbour's {index, value} entries (16 per step, 128 contiguous bytes), every lane looks its entry up in the query
// row staged in shared memory (a 8,192-bit filter first, binary search on a filter hit) and the matched products are added in
// ascending index order -- the order of the reference's block intersection (distance_impl/common.hpp:15-86) for rows with strictly
// ascending indices.  The reference's sparse "l2" is -2<x,y> (its squared norms are do_l2_distance_simd(x, x) = 0, NaN for a row
// that stores a NaN or +-inf): restated as is.
//
// HBM traffic per query (SURVEY 8d): n_dist * 4d + n_expand * 4(1+maxM0) + hops * 4(1+maxM) + 4d + 8k.
#include "hnsw_engine.h"
#include "hnsw_device.cuh"
#include "shard_merge.cuh"

#include <algorithm>
#include <atomic>
#include <cstring>

namespace pb200 {

namespace {

template <int METRIC, int STAGES, bool SPARSE>
__global__ void __launch_bounds__(256)
hnsw_search_kernel(const HnswDev ix, const float* __restrict__ Q, const HnswSparseQueries SQ, const uint32_t nq, const uint32_t efS, const uint32_t topk,
                   const uint32_t ef, uint32_t* __restrict__ out_idx, float* __restrict__ out_val, uint32_t* bitmap_all,
                   const uint32_t bitmap_words, uint32_t* vlist_all, uint2* cand_all, const uint32_t vcap, uint2* topk_all,
                   const uint32_t nbmax, const uint32_t per_warp_bytes, unsigned long long* ctrl) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const uint32_t gw = blockIdx.x * (blockDim.x >> 5) + warp;
    unsigned char* base = smem_raw + static_cast<size_t>(warp) * per_warp_bytes;
    // per-warp slice: [query | STAGES ring slots | STAGES mbarriers | neighbour ids | distances | result heap]
    // (sparse: [query indices qcap | query values qcap | filter | neighbour ids | distances | result heap])
    float* qs = reinterpret_cast<float*>(base);
    float* ring = qs + ix.vstride;
    unsigned long long* mbars = reinterpret_cast<unsigned long long*>(ring + static_cast<size_t>(STAGES) * ix.vstride);
    uint32_t* sq_idx = reinterpret_cast<uint32_t*>(base);
    float* sq_val = reinterpret_cast<float*>(sq_idx + SQ.qcap);
    uint32_t* sq_filter = reinterpret_cast<uint32_t*>(sq_val + SQ.qcap);
    uint32_t* nb_ids = SPARSE ? sq_filter + kSpFilterWords : reinterpret_cast<uint32_t*>(mbars + STAGES);
    float* nb_dist = reinterpret_cast<float*>(nb_ids + nbmax);
    uint2* topq = topk_all ? topk_all + static_cast<uint64_t>(gw) * (ef + 1) : reinterpret_cast<uint2*>(nb_dist + nbmax);
    const uint32_t mbar0 = smem_addr(mbars);
    uint32_t phase_bits = 0;
    if (STAGES > 0 && !SPARSE) {
        if (lane == 0) {
            for (int s = 0; s < STAGES; ++s) mbar_init(mbar0 + 8u * s, 1u);
            fence_proxy_async_smem();
        }
        __syncwarp();
    }
    uint32_t* bitmap = bitmap_all + static_cast<uint64_t>(gw) * bitmap_words;
    uint32_t* vlist = vlist_all + static_cast<uint64_t>(gw) * vcap;
    uint2* cand = cand_all + static_cast<uint64_t>(gw) * vcap;
    const uint32_t d = ix.feat_dim;

    for (;;) {
        unsigned long long qq = 0;
        if (lane == 0) qq = atomicAdd(&ctrl[0], 1ull);
        qq = __shfl_sync(kFull, qq, 0);
        if (qq >= nq) break;
        const uint32_t q = static_cast<uint32_t>(qq);
        unsigned long long n_dist = 0, n_expand = 0, n_hops = 0, n_entries = 0;

        SparseQuery sq{nullptr, nullptr, 0u, nullptr, false};
        if (SPARSE) {
            // stage the query row (indices, values) and the membership filter of its indices
            const unsigned long long q0 = SQ.ptr[q];
            sq.n = static_cast<uint32_t>(SQ.ptr[q + 1] - q0);
            for (uint32_t w = lane; w < kSpFilterWords; w += 32) sq_filter[w] = 0u;
            __syncwarp();
            const bool staged = sq.n <= SQ.qcap;
            bool nonfinite = false;
            for (uint32_t i = lane; i < sq.n; i += 32) {
                const uint32_t c = SQ.idx[q0 + i];
                if (staged) { sq_idx[i] = c; sq_val[i] = SQ.val[q0 + i]; }
                if (METRIC == HNSW_L2) nonfinite |= !isfinite(SQ.val[q0 + i]);
                const uint32_t h = sp_hash(c);
                atomicOr(&sq_filter[h >> 5], 1u << (h & 31u));
            }
            if (METRIC == HNSW_L2) sq.nonfinite = __any_sync(kFull, nonfinite);
            sq.idx = staged ? sq_idx : SQ.idx + q0;
            sq.val = staged ? sq_val : SQ.val + q0;
            sq.filter = sq_filter;
            __syncwarp();
        } else {
            // stage the query in the permuted layout (padding = 0)
            for (uint32_t i = lane; i < ix.vstride; i += 32) qs[i] = 0.0f;
            __syncwarp();
            const float* qrow = Q + static_cast<uint64_t>(q) * d;
            for (uint32_t i = lane; i < d; i += 32) qs[permuted_pos_dev(ix, i)] = qrow[i];
            __syncwarp();
        }
        auto distances = [&](uint32_t n) {
            if (SPARSE) batch_distances_sparse<METRIC>(ix, sq, nb_ids, nb_dist, n, lane, n_entries);
            else batch_distances<METRIC, STAGES>(ix, qs, nb_ids, nb_dist, n, lane, ring, mbar0, phase_bits);
        };

        // ---- entry point + greedy descent on levels max_level..1 (hnsw.hpp:928-959)
        uint32_t curr = ix.init_node;
        if (lane == 0) nb_ids[0] = curr;
        __syncwarp();
        distances(1);
        float curr_dist = nb_dist[0];
        n_dist += 1;
        __syncwarp();
        for (uint32_t level = ix.max_level; level >= 1; --level) {
            int changed = 1;
            while (changed) {
                changed = 0;
                const uint32_t* nb = ix.l1 + static_cast<uint64_t>(curr) * ix.l1_node_mem + static_cast<uint64_t>(level - 1) * ix.l1_level_mem;
                const uint32_t deg = min(nb[0], ix.l1_max_degree);
                n_hops += 1;
                for (uint32_t j = lane; j < deg; j += 32) nb_ids[j] = nb[1 + j];
                __syncwarp();
                if (deg) distances(deg);
                n_dist += deg;
                if (lane == 0) {
                    for (uint32_t j = 0; j < deg; ++j) {
                        const float nd = nb_dist[j];
                        if (nd < curr_dist) { curr_dist = nd; curr = nb_ids[j]; changed = 1; }
                    }
                }
                curr = __shfl_sync(kFull, curr, 0);
                curr_dist = __shfl_sync(kFull, curr_dist, 0);
                changed = __shfl_sync(kFull, changed, 0);
                __syncwarp();
            }
        }

        // ---- best-first search on level 0 (hnsw.hpp:849-924) with ef = max(efS, topk)
        int ntop = 0, ncand = 0;      // meaningful on lane 0
        uint32_t nvis = 0;            // warp-uniform
        float ub = curr_dist;         // distance(query, entry) recomputed by the reference: same value
        n_dist += 1;
        if (lane == 0) {
            heap_push<true>(topq, ntop, ub, curr);
            heap_push<false>(cand, ncand, ub, curr);
            atomicOr(&bitmap[curr >> 5], 1u << (curr & 31u));
            vlist[0] = curr;
        }
        nvis = 1;
        __syncwarp();
        int overflow = 0;
        for (;;) {
            int done = 0;
            uint32_t node = 0;
            if (lane == 0) {
                if (ncand == 0 || __uint_as_float(cand[0].x) > ub) done = 1;
                else { node = cand[0].y; heap_pop<false>(cand, ncand); }
            }
            done = __shfl_sync(kFull, done, 0);
            if (done) break;
            node = __shfl_sync(kFull, node, 0);
            const uint32_t* nb = ix.nbr0 + static_cast<uint64_t>(node) * ix.n0stride;
            const uint32_t deg = min(nb[0], ix.l0_max_degree);
            n_expand += 1;
            // A. unvisited neighbours, in list order
            uint32_t nu = 0;
            for (uint32_t b = 0; b < deg; b += 32) {
                const uint32_t j = b + lane;
                uint32_t id = 0;
                bool fresh = false;
                if (j < deg) {
                    id = nb[1 + j];
                    const uint32_t bit = 1u << (id & 31u);
                    const uint32_t old = atomicOr(&bitmap[id >> 5], bit);
                    fresh = (old & bit) == 0u;
                }
                const unsigned mask = __ballot_sync(kFull, fresh);
                if (fresh) nb_ids[nu + __popc(mask & ((1u << lane) - 1u))] = id;
                nu += __popc(mask);
            }
            __syncwarp();
            for (uint32_t i = lane; i < nu; i += 32) {
                if (nvis + i < vcap) vlist[nvis + i] = nb_ids[i];
            }
            nvis += nu;
            // B. all distances
            if (nu) distances(nu);
            n_dist += nu;
            // C. sequential replay of the queue updates (hnsw.hpp:904-914)
            if (lane == 0) {
                for (uint32_t i = 0; i < nu; ++i) {
                    const float nd = nb_dist[i];
                    if (static_cast<uint32_t>(ntop) < ef || nd < ub) {
                        if (static_cast<uint32_t>(ncand) >= vcap) { overflow = 1; break; }
                        const uint32_t id = nb_ids[i];
                        heap_push<false>(cand, ncand, nd, id);
                        heap_push<true>(topq, ntop, nd, id);
                        if (static_cast<uint32_t>(ntop) > ef) heap_pop<true>(topq, ntop);
                        if (ntop > 0) ub = __uint_as_float(topq[0].x);
                    }
                }
            }
            overflow = __shfl_sync(kFull, overflow, 0);
            if (overflow) break;
            __syncwarp();
        }
        if (overflow) {
            if (lane == 0) atomicExch(&ctrl[1], 1ull);
        }

        // ---- trim to topk and sort ascending (hnsw.hpp:961-970)
        if (lane == 0) {
            if (topk < efS) while (static_cast<uint32_t>(ntop) > topk) heap_pop<true>(topq, ntop);
            int n = ntop;
            while (n > 1) {  // std::sort_heap
                const uint2 value = topq[n - 1];
                topq[n - 1] = topq[0];
                heap_adjust<true>(topq, 0, n - 1, value);
                --n;
            }
        }
        ntop = __shfl_sync(kFull, ntop, 0);
        __syncwarp();
        for (int k = lane; k < ntop && k < static_cast<int>(topk); k += 32) {
            const uint2 e = topq[k];
            out_idx[static_cast<uint64_t>(q) * topk + k] = e.y;
            out_val[static_cast<uint64_t>(q) * topk + k] = __uint_as_float(e.x);
        }
        // ---- reset the visited bitmap for the next query of this warp
        if (nvis <= vcap) {
            for (uint32_t i = lane; i < nvis; i += 32) bitmap[vlist[i] >> 5] = 0u;
        } else {
            for (uint32_t w = lane; w < bitmap_words; w += 32) bitmap[w] = 0u;
        }
        __syncwarp();
        if (lane == 0) {
            atomicAdd(&ctrl[2], n_dist);
            atomicAdd(&ctrl[3], n_expand);
            atomicAdd(&ctrl[4], n_hops);
            atomicAdd(&ctrl[5], 1ull);
        }
        if (SPARSE) {  // per half-warp partial sums of the stored entries read
            n_entries += __shfl_xor_sync(kFull, n_entries, 16);
            if (lane == 0) atomicAdd(&ctrl[6], n_entries);
        }
    }
}

// Index sharding: this shard's [nq][topk] search results -> exchange records.  An empty slot (out_idx == 0xFFFFFFFF, the fill
// of the sharded path) gets key 0.  key = (~o << 32) | ~(rank * topk + slot) with o = orderable(dist), and o = 0xFFFFFFFF for
// every NaN whatever its sign and payload: the merge orders by distance ascending with NaN last, then shard rank, then slot,
// so one shard's own order (ties included) is kept wherever it is sorted -- a NaN in the search heaps can leave it out of order,
// and the merge sorts it; the low word is never 0 while (rank + 1) * topk <= kSelKeys.
__global__ void hnsw_shard_pack_kernel(const uint32_t* __restrict__ idx, const float* __restrict__ val, const uint64_t n,
                                       const uint32_t topk, const uint32_t rank, const uint32_t id_offset,
                                       ShardRecord* __restrict__ rec) {
    const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t slot = static_cast<uint32_t>(i % topk);
    const uint32_t id = idx[i];
    ShardRecord out{0ull, 0u, 0.0f};
    if (id != 0xFFFFFFFFu) {
        const float d = val[i];
        const uint32_t o = isnan(d) ? 0xFFFFFFFFu : orderable(d);
        out.key = (static_cast<unsigned long long>(~o) << 32) | static_cast<unsigned long long>(~(rank * topk + slot));
        out.id = id_offset + id;
        out.val = d;
    }
    rec[i] = out;
}

constexpr uint64_t kStageBytes = 32ull << 20;  // pinned staging of base rows and neighbour lists, per chunk

// Copies rows [0, n) to dst through pinned staging memory: row r takes elements [off(r), off(r + 1)) of dst, and fill(r, out)
// writes all of them, padding included, to `out`.  Chunks of whole rows of at most kStageBytes (a longer row: alone).
template <typename T, typename Off, typename Fill>
void stage_rows(T* dst, uint64_t n, const Off& off, const Fill& fill, cudaStream_t stream) {
    PinnedBuffer<T> buf;  // sized once: chunks vary in size, and re-pinning costs more than the copy (grows only for a longer row)
    buf.reserve(std::max<uint64_t>(1, std::min<uint64_t>(off(n) - off(0), kStageBytes / sizeof(T))));
    for (uint64_t c0 = 0; c0 < n;) {
        uint64_t c1 = c0 + 1, hi = n;  // the most rows from c0 on that fit, at least one
        while (c1 < hi) {
            const uint64_t mid = (c1 + hi + 1) / 2;
            if ((off(mid) - off(c0)) * sizeof(T) <= kStageBytes) c1 = mid; else hi = mid - 1;
        }
        const uint64_t e0 = off(c0), en = off(c1) - e0;
        buf.reserve(std::max<uint64_t>(en, 1));
        parallel_for_chunks(c1 - c0, [&](uint64_t r) { fill(c0 + r, buf.get() + (off(c0 + r) - e0)); });
        if (en) PB200_CUDA(cudaMemcpyAsync(dst + e0, buf.get(), en * sizeof(T), cudaMemcpyHostToDevice, stream));
        PB200_CUDA(cudaStreamSynchronize(stream));
        c0 = c1;
    }
}

void check_shard_slots(uint32_t rank, uint32_t topk) {
    if ((static_cast<uint64_t>(rank) + 1) * topk > static_cast<uint64_t>(kSelKeys))
        throw std::runtime_error("pecos_b200: (rank + 1) * topk exceeds the shard merge capacity of 1024 records per query");
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------------
uint32_t warp_smem_bytes(bool sparse, uint32_t vstride, int stages, uint32_t qcap, uint32_t tail) {
    const uint32_t query = sparse ? qcap * 8u + kSpFilterWords * 4u
                                  : vstride * 4u * (1u + static_cast<uint32_t>(stages)) + static_cast<uint32_t>(stages) * 8u;
    return (query + tail + 15u) & ~15u;
}

HnswPlan hnsw_plan(bool sparse, uint32_t vstride, uint32_t max_degree, int stages, uint32_t ef, uint32_t qcap) {
    const uint32_t nbmax = ((max_degree + 31u) / 32u) * 32u;
    HnswPlan p{false, 0, false, 0u, nbmax};
    for (const bool heap_in_smem : {true, false}) {
        if (heap_in_smem && ef > kEfSmemMax) continue;
        const uint32_t tail = nbmax * 8u + (heap_in_smem ? (ef + 1u) * 8u : 0u);
        for (int s = sparse ? 0 : (stages <= 0 ? 0 : (stages <= 4 ? 4 : 8));; s = s > 4 ? 4 : 0) {
            p = HnswPlan{false, s, heap_in_smem, warp_smem_bytes(sparse, vstride, s, qcap, tail), nbmax};
            if (p.per_warp <= kWarpSmemMax) { p.fits = true; return p; }
            if (s == 0) break;
        }
    }
    return p;
}

CtaShape cta_shape(int device, uint32_t per_warp, uint32_t max_warps_per_sm) {
    uint32_t warps = 8;
    while (warps > 1 && static_cast<uint64_t>(warps) * per_warp > 96u * 1024u) warps >>= 1;
    int sms = 132;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    const uint32_t by_smem = static_cast<uint32_t>((220u * 1024u) / (static_cast<uint64_t>(warps) * per_warp));
    return CtaShape{warps, std::max<uint32_t>(1, std::min<uint32_t>(max_warps_per_sm / warps, by_smem)), static_cast<uint32_t>(sms)};
}

void DeviceQueries::upload(const HostMatrix& x, uint32_t rows, cudaStream_t stream) {
    std::vector<unsigned long long> ptr;
    if (!x.row_ptr) {
        val_.upload(x.dense, static_cast<uint64_t>(rows) * x.cols, stream);
        qcap_ = 0;
    } else {
        const uint64_t e0 = x.row_ptr[0], nnz = x.row_ptr[rows] - e0;
        ptr.resize(static_cast<size_t>(rows) + 1);
        uint64_t longest = 0;
        for (uint32_t i = 0; i <= rows; ++i) {
            ptr[i] = x.row_ptr[i] - e0;
            if (i) longest = std::max<uint64_t>(longest, x.row_ptr[i] - x.row_ptr[i - 1]);
        }
        ptr_.upload(ptr.data(), ptr.size(), stream);
        idx_.reserve(std::max<uint64_t>(nnz, 1));
        val_.reserve(std::max<uint64_t>(nnz, 1));
        if (nnz) {
            PB200_CUDA(cudaMemcpyAsync(idx_.get(), x.col_idx + e0, nnz * 4, cudaMemcpyHostToDevice, stream));
            PB200_CUDA(cudaMemcpyAsync(val_.get(), x.val + e0, nnz * 4, cudaMemcpyHostToDevice, stream));
        }
        qcap_ = static_cast<uint32_t>(std::min<uint64_t>(kSpQcapMax, (std::max<uint64_t>(longest, 1) + 31) / 32 * 32));
    }
    PB200_CUDA(cudaStreamSynchronize(stream));  // `ptr` is a local, and the caller may release x on return
}

uint64_t DeviceRows::upload(uint64_t n, uint32_t feat_dim, bool sparse, const RowFn& row, cudaStream_t stream, HnswDev* view) {
    if (sparse) {
        std::vector<unsigned long long> ptr(n + 1, 0ull);
        for (uint64_t r = 0; r < n; ++r) {
            const float* v; const uint32_t* c;
            ptr[r + 1] = ptr[r] + row(r, &v, &c);
        }
        const uint64_t nnz = ptr[n];
        sp_ptr_.upload(ptr.data(), n + 1, stream);
        sp_ent_.reserve(std::max<uint64_t>(nnz, 1));
        stage_rows(sp_ent_.get(), n, [&](uint64_t r) { return ptr[r]; }, [&](uint64_t r, uint2* dst) {
            const float* v; const uint32_t* c;
            const uint32_t len = row(r, &v, &c);
            for (uint32_t j = 0; j < len; ++j) {
                uint32_t bits;
                std::memcpy(&bits, v + j, 4);
                dst[j] = make_uint2(c[j], bits);
            }
        }, stream);
        PB200_CUDA(cudaStreamSynchronize(stream));  // `ptr` is a local
        view->sp_ptr = sp_ptr_.get();
        view->sp_ent = sp_ent_.get();
        return (n + 1) * 8 + nnz * 8;
    }
    const uint32_t vs = dense_vstride(feat_dim);
    std::vector<uint32_t> pos(feat_dim);
    for (uint32_t i = 0; i < feat_dim; ++i) pos[i] = dense_permuted_pos(feat_dim, i);
    vec_.reserve(std::max<uint64_t>(n * vs, 1));
    stage_rows(vec_.get(), n, [vs](uint64_t r) { return r * vs; }, [&](uint64_t r, float* dst) {
        const float* v; const uint32_t* c;
        row(r, &v, &c);
        std::fill(dst, dst + vs, 0.0f);
        for (uint32_t i = 0; i < feat_dim; ++i) dst[pos[i]] = v[i];
    }, stream);
    view->vec = vec_.get();
    view->vstride = vs;
    view->main_pad = dense_main_pad(feat_dim);
    view->tail_len = dense_tail_len(feat_dim);
    return n * vs * 4;
}

HnswEngine::HnswEngine(std::unique_ptr<HnswHostIndex> host, int device) : host_(std::move(host)), device_(device) {
    PB200_CUDA(cudaSetDevice(device_));
    PB200_CUDA(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    for (auto& e : ev_) PB200_CUDA(cudaEventCreate(&e));
    const HnswHostIndex& H = *host_;
    const uint64_t N = H.num_node;
    const uint32_t n0 = H.n0stride();
    index_bytes_ = rows_.upload(N, H.feat_dim, H.sparse, [&H](uint64_t r, const float** v, const uint32_t** c) {
        const uint32_t node = static_cast<uint32_t>(r);
        if (H.sparse) return H.l0_sparse_row(node, v, c);
        *v = H.l0_vector(node);
        return H.feat_dim;
    }, stream_, &view_);
    nbr0_.reserve(N * n0);
    stage_rows(nbr0_.get(), N, [n0](uint64_t r) { return r * n0; }, [&H, n0](uint64_t r, uint32_t* nd) {
        const uint32_t* nb = H.l0_neighborhood(static_cast<uint32_t>(r));
        const uint32_t deg = std::min(nb[0], H.l0_max_degree);
        std::fill(nd, nd + n0, 0u);
        nd[0] = deg;
        for (uint32_t j = 0; j < deg; ++j) nd[1 + j] = nb[1 + j];
    }, stream_);
    uint64_t l1_len = 0;
    if (H.max_level > 0) {
        l1_len = static_cast<uint64_t>(N) * H.l1_node_mem_size;
        l1_.upload(H.l1_buffer, l1_len, stream_);
        PB200_CUDA(cudaStreamSynchronize(stream_));
    }
    index_bytes_ += N * n0 * 4 + l1_len * 4;
    view_.nbr0 = nbr0_.get();
    view_.l1 = l1_.get();
    view_.num_node = H.num_node;
    view_.max_level = H.max_level;
    view_.init_node = H.init_node;
    view_.feat_dim = H.feat_dim;
    view_.n0stride = n0;
    view_.l0_max_degree = H.l0_max_degree;
    view_.l1_node_mem = H.l1_node_mem_size;
    view_.l1_level_mem = H.l1_level_mem_size;
    view_.l1_max_degree = H.l1_max_degree;
    view_.metric = H.metric;
    ctrl_.reserve(8);
    PB200_CUDA(cudaMemsetAsync(ctrl_.get(), 0, 8 * sizeof(unsigned long long), stream_));
    PB200_CUDA(cudaStreamSynchronize(stream_));
    const int max_smem = static_cast<int>(kWarpSmemMax);
    PB200_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<HNSW_IP, 0, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<HNSW_L2, 0, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<HNSW_IP, 4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<HNSW_L2, 4, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<HNSW_IP, 8, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<HNSW_L2, 8, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<HNSW_IP, 0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(hnsw_search_kernel<HNSW_L2, 0, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    stages_ = 4;  // rows in flight per warp through the bulk-copy ring; 0 = direct loads (first-generation kernel)
    if (const char* env = std::getenv("PB200_HNSW_STAGES")) {
        const int v = std::atoi(env);
        stages_ = (v <= 0) ? 0 : (v <= 4 ? 4 : 8);
    }
    // the mapped file is no longer needed once the arrays live in HBM
    host_->l0_buffer = nullptr;
    host_->l0_mem_start = nullptr;
    host_->l1_buffer = nullptr;
    host_->store.reset();
}

HnswEngine::~HnswEngine() {
    cudaSetDevice(device_);
    if (stream_) cudaStreamSynchronize(stream_);
    for (auto& e : ev_) if (e) cudaEventDestroy(e);
    if (stream_) cudaStreamDestroy(stream_);
}

HnswPlan HnswEngine::plan_(uint32_t ef, uint32_t qcap) const {
    const HnswHostIndex& H = *host_;
    return hnsw_plan(H.sparse, view_.vstride, std::max(H.l0_max_degree, H.l1_max_degree), stages_, ef, qcap);
}

HnswPlan HnswEngine::search_plan(uint32_t efS, uint32_t topk) const {
    return plan_(std::max(efS, topk), host_->sparse ? kSpQcapMax : 0u);
}

void HnswEngine::set_stages(int stages) {
    stages_ = (stages <= 0) ? 0 : (stages <= 4 ? 4 : 8);
    n_warps_ = 0;  // forces the scratch / launch geometry to be recomputed
}

// One warp's shared-memory slice must fit kWarpSmemMax.  The ring takes stages + 1 rows of 4 * vstride bytes, so wide vectors
// run the deepest ring that fits, and the widest ones move the result heap to global memory too (hnsw_plan).  Results do not
// depend on the plan.  Callers check search_plan first (HNSW.predict raises ValueError), so the throw is a last guard.
void HnswEngine::ensure_scratch_(uint32_t ef, uint32_t qcap) {
    const HnswHostIndex& H = *host_;
    const HnswPlan plan = plan_(ef, qcap);
    if (!plan.fits)
        throw std::runtime_error("pecos_b200: HNSW query dimension too large for the shared-memory staging area, even with "
                                 "direct loads and the result heap in global memory");
    run_plan_ = plan;
    const bool top_in_smem = plan.heap_in_smem;
    const uint32_t per_warp = plan.per_warp;
    const CtaShape shape = cta_shape(device_, per_warp, H.sparse ? 32u : 16u);
    const uint32_t warps = shape.warps, sms = shape.sms;
    uint32_t n_ctas = sms * shape.ctas_per_sm;
    // bound the scratch footprint (bitmap N/8 bytes per warp)
    const uint64_t words = (static_cast<uint64_t>(H.num_node) + 31) / 32;
    uint32_t vcap = 32768;
    if (const char* env = std::getenv("PB200_HNSW_VCAP")) vcap = static_cast<uint32_t>(std::max<uint64_t>(64, std::strtoull(env, nullptr, 10)));
    vcap = std::max(vcap, vcap_floor_);  // raised by launch_ after a candidate-queue overflow
    vcap = static_cast<uint32_t>(std::min<uint64_t>(vcap, static_cast<uint64_t>(H.num_node) + 1));
    const uint64_t per_warp_scratch = words * 4 + static_cast<uint64_t>(vcap) * 12 + (top_in_smem ? 0 : static_cast<uint64_t>(ef + 1) * 8);
    while (n_ctas > sms && static_cast<uint64_t>(n_ctas) * warps * per_warp_scratch > (24ull << 30)) n_ctas -= sms;
    const uint32_t n_warps = n_ctas * warps;
    if (n_warps != n_warps_ || vcap != vcap_ || warps != warps_per_cta_) {
        bitmap_.reserve(static_cast<uint64_t>(n_warps) * words);
        PB200_CUDA(cudaMemsetAsync(bitmap_.get(), 0, static_cast<uint64_t>(n_warps) * words * 4, stream_));
        vlist_.reserve(static_cast<uint64_t>(n_warps) * vcap);
        cand_.reserve(static_cast<uint64_t>(n_warps) * vcap);
        n_warps_ = n_warps; warps_per_cta_ = warps; n_ctas_ = n_ctas; vcap_ = vcap;
    }
    // grows only: kept across calls, sized for this call's warps and ef whatever the calls in between used
    if (!top_in_smem) topk_heap_.reserve(static_cast<uint64_t>(n_warps) * (ef + 1));
}

void HnswEngine::launch_info(uint64_t* out) const {
    out[0] = static_cast<uint64_t>(run_plan_.stages);
    out[1] = warps_per_cta_;
    out[2] = last_ctas_;
    out[3] = last_smem_;
    out[4] = topk_heap_.capacity();
}

double HnswEngine::launch_once_(const SearchIo& io, uint32_t efS, uint32_t topk, int idx_fill, bool* overflow) {
    const HnswHostIndex& H = *host_;
    const uint32_t ef = std::max(efS, topk), nq = io.nq;
    if (ef == 0) throw std::runtime_error("pecos_b200: efS and topk are both zero");
    ensure_scratch_(ef, io.queries->qcap());
    const uint32_t nbmax = run_plan_.nbmax, per_warp = run_plan_.per_warp;
    const bool top_in_smem = run_plan_.heap_in_smem;
    const int stages = run_plan_.stages;
    const uint32_t words = static_cast<uint32_t>((static_cast<uint64_t>(H.num_node) + 31) / 32);
    PB200_CUDA(cudaMemsetAsync(ctrl_.get(), 0, 8 * sizeof(unsigned long long), stream_));
    PB200_CUDA(cudaMemsetAsync(io.idx, idx_fill, static_cast<uint64_t>(nq) * topk * 4, stream_));
    PB200_CUDA(cudaMemsetAsync(io.val, 0, static_cast<uint64_t>(nq) * topk * 4, stream_));
    const uint32_t ctas = std::max<uint32_t>(1, std::min<uint32_t>(n_ctas_, (nq + warps_per_cta_ - 1) / warps_per_cta_));
    const size_t smem = static_cast<size_t>(warps_per_cta_) * per_warp;
    const float* q_dev = io.queries->dense();
    const HnswSparseQueries sq = io.queries->sparse();
    PB200_CUDA(cudaEventRecord(ev_[0], stream_));
    auto launch = [&](auto kernel) {
        kernel<<<ctas, warps_per_cta_ * 32, smem, stream_>>>(view_, q_dev, sq, nq, efS, topk, ef, io.idx, io.val,
                                                             bitmap_.get(), words, vlist_.get(), cand_.get(), vcap_,
                                                             top_in_smem ? nullptr : topk_heap_.get(), nbmax, per_warp, ctrl_.get());
    };
    const bool ip = H.metric == HNSW_IP;
    if (H.sparse) { if (ip) launch(hnsw_search_kernel<HNSW_IP, 0, true>); else launch(hnsw_search_kernel<HNSW_L2, 0, true>); }
    else if (stages == 0) { if (ip) launch(hnsw_search_kernel<HNSW_IP, 0, false>); else launch(hnsw_search_kernel<HNSW_L2, 0, false>); }
    else if (stages == 4) { if (ip) launch(hnsw_search_kernel<HNSW_IP, 4, false>); else launch(hnsw_search_kernel<HNSW_L2, 4, false>); }
    else { if (ip) launch(hnsw_search_kernel<HNSW_IP, 8, false>); else launch(hnsw_search_kernel<HNSW_L2, 8, false>); }
    PB200_CUDA(cudaGetLastError());
    last_ctas_ = ctas;
    last_smem_ = static_cast<uint32_t>(smem);
    PB200_CUDA(cudaEventRecord(ev_[1], stream_));
    ++launches_;
    PB200_CUDA(cudaEventSynchronize(ev_[1]));
    float ms = 0.f;
    PB200_CUDA(cudaEventElapsedTime(&ms, ev_[0], ev_[1]));
    unsigned long long flag[2] = {0, 0};
    PB200_CUDA(cudaMemcpy(flag, ctrl_.get(), sizeof(flag), cudaMemcpyDeviceToHost));
    *overflow = flag[1] != 0;
    last_ms_ = ms;
    return ms;
}

// A query whose candidate queue outgrows the per-warp scratch (vcap entries) flags an overflow; the batch is then re-run with
// twice the capacity (at most num_node + 1 entries, which can never overflow: a node enters the queue at most once), instead
// of aborting the host process.
double HnswEngine::launch_(const SearchIo& io, uint32_t efS, uint32_t topk, int idx_fill) {
    for (;;) {
        bool overflow = false;
        const double ms = launch_once_(io, efS, topk, idx_fill, &overflow);
        if (!overflow) return ms;
        const uint64_t cap_max = static_cast<uint64_t>(host_->num_node) + 1;
        if (vcap_ >= cap_max) throw std::runtime_error("pecos_b200: HNSW candidate queue overflow at full capacity (internal error)");
        vcap_floor_ = static_cast<uint32_t>(std::min<uint64_t>(cap_max, static_cast<uint64_t>(vcap_) * 2));
        ++vcap_retries_;
    }
}


bool HnswEngine::upload_(const HostMatrix& x, uint32_t topk, DeviceQueries& into) {
    PB200_CUDA(cudaSetDevice(device_));
    if (host_->sparse && !x.row_ptr) throw std::runtime_error("pecos_b200: dense queries against a sparse (csr) HNSW index");
    if (!host_->sparse && x.row_ptr) throw std::runtime_error("pecos_b200: csr queries against a dense HNSW index");
    if (x.cols != host_->feat_dim) throw std::runtime_error("pecos_b200: query dimension != index dimension");
    if (x.rows == 0 || topk == 0) return false;
    into.upload(x, x.rows, stream_);
    return true;
}

void HnswEngine::predict(const HostMatrix& x, uint32_t efS, uint32_t topk, uint32_t* ret_idx, float* ret_val) {
    if (!upload_(x, topk, queries_)) return;
    const uint64_t n = static_cast<uint64_t>(x.rows) * topk;
    out_idx_.reserve(n);
    out_val_.reserve(n);
    launch_({&queries_, x.rows, out_idx_.get(), out_val_.get()}, efS, topk);
    // rows with fewer than topk results keep the caller's zeros (libpecos.cpp:554-558): our buffers were zeroed too
    PB200_CUDA(cudaMemcpyAsync(ret_idx, out_idx_.get(), n * 4, cudaMemcpyDeviceToHost, stream_));
    PB200_CUDA(cudaMemcpyAsync(ret_val, out_val_.get(), n * 4, cudaMemcpyDeviceToHost, stream_));
    PB200_CUDA(cudaStreamSynchronize(stream_));
}

void HnswEngine::resident_upload(const HostMatrix& x) {
    res_nq_ = 0;
    upload_(x, 1, res_queries_);  // searched later with resident_predict's topk
    res_nq_ = x.rows;
}

double HnswEngine::resident_predict(uint32_t efS, uint32_t topk) {
    PB200_CUDA(cudaSetDevice(device_));
    if (!res_nq_) throw std::runtime_error("pecos_b200: no resident query batch uploaded");
    res_idx_.reserve(static_cast<uint64_t>(res_nq_) * topk);
    res_val_.reserve(static_cast<uint64_t>(res_nq_) * topk);
    res_topk_ = topk;
    return launch_({&res_queries_, res_nq_, res_idx_.get(), res_val_.get()}, efS, topk);
}

void HnswEngine::resident_fetch(uint32_t* ret_idx, float* ret_val) {
    PB200_CUDA(cudaSetDevice(device_));
    PB200_CUDA(cudaMemcpy(ret_idx, res_idx_.get(), static_cast<uint64_t>(res_nq_) * res_topk_ * 4, cudaMemcpyDeviceToHost));
    PB200_CUDA(cudaMemcpy(ret_val, res_val_.get(), static_cast<uint64_t>(res_nq_) * res_topk_ * 4, cudaMemcpyDeviceToHost));
}

// search into out_idx_ / out_val_ (empty slots 0xFFFFFFFF), then pack the records into the caller's device buffer
void HnswEngine::sharded_local_packed(const HostMatrix& x, uint32_t efS, uint32_t topk, uint32_t rank, uint32_t id_offset,
                                      void* rec_dev) {
    check_shard_slots(rank, topk);
    if (!upload_(x, topk, queries_)) return;
    const uint64_t n = static_cast<uint64_t>(x.rows) * topk;
    out_idx_.reserve(n);
    out_val_.reserve(n);
    launch_({&queries_, x.rows, out_idx_.get(), out_val_.get()}, efS, topk, 0xFF);
    hnsw_shard_pack_kernel<<<static_cast<uint32_t>((n + 255) / 256), 256, 0, stream_>>>(out_idx_.get(), out_val_.get(), n, topk, rank,
                                                                                      id_offset, static_cast<ShardRecord*>(rec_dev));
    PB200_CUDA(cudaGetLastError());
    ++launches_;
    PB200_CUDA(cudaStreamSynchronize(stream_));
}

void HnswEngine::sharded_merge_packed(uint32_t world, uint32_t rows, uint32_t topk, const void* g_rec, uint32_t* ret_idx,
                                      float* ret_val) {
    PB200_CUDA(cudaSetDevice(device_));
    if (world == 0) throw std::runtime_error("pecos_b200: world must be >= 1");
    if (static_cast<uint64_t>(world) * topk > static_cast<uint64_t>(kSelKeys))
        throw std::runtime_error("pecos_b200: world * topk exceeds the shard merge capacity of 1024 records per query");
    if (rows == 0 || topk == 0) return;
    const uint64_t n = static_cast<uint64_t>(rows) * topk;
    out_idx_.reserve(n);
    out_val_.reserve(n);
    merge_cnt_.reserve(rows);
    // the merge writes each row's first min(topk, records) entries; the tail keeps these zeros (libpecos.cpp:554-558)
    PB200_CUDA(cudaMemsetAsync(out_idx_.get(), 0, n * 4, stream_));
    PB200_CUDA(cudaMemsetAsync(out_val_.get(), 0, n * 4, stream_));
    shard_merge_packed_kernel<<<(rows + kSelWarps - 1) / kSelWarps, kSelWarps * 32, 0, stream_>>>(
        static_cast<const ShardRecord*>(g_rec), world, rows, topk, topk, out_idx_.get(), out_val_.get(), merge_cnt_.get());
    PB200_CUDA(cudaGetLastError());
    ++launches_;
    PB200_CUDA(cudaMemcpyAsync(ret_idx, out_idx_.get(), n * 4, cudaMemcpyDeviceToHost, stream_));
    PB200_CUDA(cudaMemcpyAsync(ret_val, out_val_.get(), n * 4, cudaMemcpyDeviceToHost, stream_));
    PB200_CUDA(cudaStreamSynchronize(stream_));
}

HnswCounters HnswEngine::counters() {
    PB200_CUDA(cudaSetDevice(device_));
    unsigned long long h[8];
    PB200_CUDA(cudaMemcpy(h, ctrl_.get(), sizeof(h), cudaMemcpyDeviceToHost));
    HnswCounters c;
    c.n_dist = h[2]; c.n_expand = h[3]; c.n_hops = h[4]; c.n_queries = h[5]; c.n_entries = h[6];
    return c;
}

}  // namespace pb200
