// Host-side HNSW index ingest: <model>/c_model/{config.json,index.mmap_store} -> arrays re-laid-out for HBM.
//
// Reference behaviour restated here:
//   HNSW::load / load_config ....... pecos/core/ann/hnsw.hpp:470-488, :534-552
//   GraphL0 record layout .......... pecos/core/ann/hnsw.hpp:92-178   [deg u32][max_degree x u32][len u32][d x f32]
//   GraphL1 layout ................. pecos/core/ann/hnsw.hpp:180-220
//   container ...................... pecos/core/utils/mmap_util.hpp (read side: host_io.h MmapStoreReader)
//
// HBM layout (ours):
//   vec[N][vstride]   float32, the first 16*floor(d/16) components PERMUTED so that a half-warp's 16 lanes each read one
//                     float4 per 64 components and lane j receives, in order, exactly the components the reference's
//                     avx512 kernel accumulates in SIMD lane j (component 16k+j -> position 64*(k/4) + 4*j + k%4);
//                     zero-padded to a multiple of 64; the remaining d%16 components follow in natural order, padded
//                     to 16.  Rows are 16-byte aligned (the reference's records are not: SURVEY 7.3-9).
//   nbr0[N][n0stride] uint32 {deg, ids...} of level 0, stride padded to a multiple of 4
//   l1[...]           the reference's upper-level buffer, verbatim
//
// Sparse (csr) indices -- HNSW<float, FeatVecSparse{IP,L2}Simd<uint32_t, float>> (libpecos.cpp:449-450): level-0 records are
// variable-sized, [deg u32][max_degree x u32][len u32][len x f32 values][len x u32 indices] at byte offset mem_start_of_node[node]
// (feat_vectors.hpp:97-131, hnsw.hpp:122-176).  HBM layout: sp_ptr[N+1] entry offsets + sp_ent[nnz] interleaved {index, value bits}
// (one coalesced 8-byte stream per row), nbr0 as above.
#pragma once

#include <algorithm>
#include <thread>

#include "host_io.h"

namespace pb200 {

enum HnswMetric { HNSW_IP = 0, HNSW_L2 = 1 };

// The dense device row layout above, for rows of d components: the permuted main part, its padded length, the natural-order
// tail and the row stride (floats)
inline uint32_t dense_len16(uint32_t d) { return d / 16u; }
inline uint32_t dense_main_pad(uint32_t d) { return 64u * ((dense_len16(d) + 3u) / 4u); }
inline uint32_t dense_tail_len(uint32_t d) { return d - 16u * dense_len16(d); }
inline uint32_t dense_vstride(uint32_t d) { return dense_main_pad(d) + (dense_tail_len(d) ? 16u : 0u); }
// component i of a d-component vector -> position inside its dense_vstride(d)-long device row
inline uint32_t dense_permuted_pos(uint32_t d, uint32_t i) {
    const uint32_t m = 16u * dense_len16(d);
    if (i < m) {
        const uint32_t k = i / 16u, j = i % 16u;
        return 64u * (k / 4u) + 4u * j + (k % 4u);
    }
    return dense_main_pad(d) + (i - m);
}

struct HnswHostIndex {
    uint32_t num_node = 0, maxM = 0, maxM0 = 0, efC = 0, max_level = 0, init_node = 0;
    uint32_t feat_dim = 0;
    int metric = HNSW_IP;
    bool sparse = false;                    // FeatVecSparse records (variable size)
    const uint64_t* l0_mem_start = nullptr;  // [num_node + 1] byte offsets into l0_buffer (sparse)
    // views into the mapped file
    std::unique_ptr<MmapStoreReader> store;
    const uint8_t* l0_buffer = nullptr;
    uint64_t l0_buffer_size = 0;
    uint32_t l0_max_degree = 0, l0_node_mem_size = 0;
    const uint32_t* l1_buffer = nullptr;
    uint64_t l1_buffer_len = 0;
    uint32_t l1_max_level = 0, l1_max_degree = 0, l1_node_mem_size = 0, l1_level_mem_size = 0;

    uint32_t n0stride() const { return (1u + l0_max_degree + 3u) & ~3u; }

    const uint32_t* l0_neighborhood(uint32_t node) const {
        return reinterpret_cast<const uint32_t*>(l0_buffer + (sparse ? l0_mem_start[node] : static_cast<uint64_t>(node) * l0_node_mem_size));
    }
    // sparse record of a node: number of stored entries, its values and (ascending) indices
    uint32_t l0_sparse_row(uint32_t node, const float** val, const uint32_t** idx) const {
        const uint8_t* fv = l0_buffer + l0_mem_start[node] + static_cast<uint64_t>(1 + l0_max_degree) * 4;
        const uint32_t len = *reinterpret_cast<const uint32_t*>(fv);
        *val = reinterpret_cast<const float*>(fv + 4);
        *idx = reinterpret_cast<const uint32_t*>(fv + 4 + static_cast<uint64_t>(len) * 4);
        return len;
    }
    const float* l0_vector(uint32_t node) const {
        return reinterpret_cast<const float*>(l0_buffer + static_cast<uint64_t>(node) * l0_node_mem_size +
                                              static_cast<uint64_t>(1 + l0_max_degree) * 4 + 4);
    }
};

inline const char* hnsw_type_name(int metric, bool sparse = false) {
    if (sparse)
        return metric == HNSW_IP ? "pecos::ann::HNSW<float, pecos::ann::FeatVecSparseIPSimd<uint32_t, float>>"
                                 : "pecos::ann::HNSW<float, pecos::ann::FeatVecSparseL2Simd<uint32_t, float>>";
    return metric == HNSW_IP ? "pecos::ann::HNSW<float, pecos::ann::FeatVecDenseIPSimd<float>>"
                             : "pecos::ann::HNSW<float, pecos::ann::FeatVecDenseL2Simd<float>>";
}

inline std::unique_ptr<HnswHostIndex> load_hnsw_index(const std::string& model_dir, int metric, bool lazy_load, bool sparse = false) {
    JsonValue cfg = json_parse_file(model_dir + "/config.json");
    const std::string want = hnsw_type_name(metric, sparse);
    const JsonValue* t = cfg.find("hnsw_t");
    const std::string got = (t && t->kind == JsonValue::String) ? t->str : std::string("<missing>");
    if (got != want) throw std::invalid_argument("Inconsistent HNSW_T: hnsw_t_cur = " + want + " hnsw_t_inp = " + got);
    const JsonValue* v = cfg.find("version");
    const std::string version = (v && v->kind == JsonValue::String) ? v->str : std::string("not found");
    if (version != "v2.0") throw std::runtime_error("Unable to load memory-mapped file with version = " + version);

    auto idx = std::make_unique<HnswHostIndex>();
    idx->metric = metric;
    idx->sparse = sparse;
    idx->store = std::make_unique<MmapStoreReader>(model_dir + "/index.mmap_store", lazy_load);
    MmapStoreReader& s = *idx->store;
    idx->num_node = s.get_one<uint32_t>();
    idx->maxM = s.get_one<uint32_t>();
    idx->maxM0 = s.get_one<uint32_t>();
    idx->efC = s.get_one<uint32_t>();
    idx->max_level = s.get_one<uint32_t>();
    idx->init_node = s.get_one<uint32_t>();
    // GraphL0::load (hnsw.hpp:113-120)
    const uint32_t l0_nodes = s.get_one<uint32_t>();
    idx->feat_dim = s.get_one<uint32_t>();
    idx->l0_max_degree = s.get_one<uint32_t>();
    idx->l0_node_mem_size = s.get_one<uint32_t>();
    uint64_t n_starts = 0;
    idx->l0_mem_start = s.get_vector<uint64_t>(&n_starts);
    idx->l0_buffer = reinterpret_cast<const uint8_t*>(s.get_vector<char>(&idx->l0_buffer_size));
    // GraphL1::load (hnsw.hpp:197-204)
    const uint32_t l1_nodes = s.get_one<uint32_t>();
    idx->l1_max_level = s.get_one<uint32_t>();
    idx->l1_max_degree = s.get_one<uint32_t>();
    idx->l1_node_mem_size = s.get_one<uint32_t>();
    idx->l1_level_mem_size = s.get_one<uint32_t>();
    idx->l1_buffer = s.get_vector<uint32_t>(&idx->l1_buffer_len);

    if (l0_nodes != idx->num_node || l1_nodes != idx->num_node) throw std::runtime_error("hnsw index: node counts disagree");
    if (sparse) {
        if (n_starts != static_cast<uint64_t>(idx->num_node) + 1 || idx->l0_mem_start[idx->num_node] != idx->l0_buffer_size)
            throw std::runtime_error("hnsw index: level-0 record offsets do not match the buffer (not a sparse float32 index?)");
        const uint64_t head = static_cast<uint64_t>(1 + idx->l0_max_degree) * 4 + 4;
        for (uint32_t i = 0; i < idx->num_node; ++i) {
            const uint64_t b = idx->l0_mem_start[i], e = idx->l0_mem_start[i + 1];
            if (e < b + head || e > idx->l0_buffer_size) throw std::runtime_error("hnsw index: bad level-0 record offsets");
            const uint32_t len = *reinterpret_cast<const uint32_t*>(idx->l0_buffer + b + head - 4);
            if (e - b != head + static_cast<uint64_t>(len) * 8) throw std::runtime_error("hnsw index: level-0 record size mismatch");
        }
    } else {
        const uint64_t rec = static_cast<uint64_t>(1 + idx->l0_max_degree) * 4 + 4 + static_cast<uint64_t>(idx->feat_dim) * 4;
        if (idx->l0_node_mem_size != rec) throw std::runtime_error("hnsw index: unexpected level-0 record size (not a dense float32 index?)");
        if (idx->l0_buffer_size != rec * idx->num_node) throw std::runtime_error("hnsw index: level-0 buffer size mismatch");
    }
    if (idx->max_level > 0 && idx->l1_buffer_len < static_cast<uint64_t>(idx->num_node) * idx->l1_node_mem_size)
        throw std::runtime_error("hnsw index: level>=1 buffer too small");
    if (idx->num_node == 0 || idx->init_node >= idx->num_node) throw std::runtime_error("hnsw index: bad init_node");
    return idx;
}

}  // namespace pb200
