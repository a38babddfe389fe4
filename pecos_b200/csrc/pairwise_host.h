// Host side of PairwiseANN: the model's arrays in host memory, the reader of <c_model>/{config.json,index.mmap_store} and the
// writer of the same folder.
//
// Reference behaviour restated here:
//   PairwiseANN::train ............. pecos/core/ann/pairwise.hpp:245-263   (deep copy of X_trn and Y_csc)
//   PairwiseANN::save / load ....... pecos/core/ann/pairwise.hpp:206-243
//   save_mat / load_mat ............ pecos/core/ann/pairwise.hpp:60-102
//   save_config / load_config ...... pecos/core/ann/pairwise.hpp:158-204   (nlohmann::json dump(4): keys in sorted order)
//
// index.mmap_store blocks, in order: N, L, d (u32 each); Y_csc as {rows u32, cols u32, nnz u64, col_ptr u64[L+1],
// row_idx u32[nnz], val f32[nnz]}; X_trn as the same csr record (row_ptr u64[N+1]) or, dense, {rows, cols, nnz = N*d, val f32[nnz]}.
#pragma once

#include <sys/stat.h>

#include <cerrno>
#include <cstdio>
#include <memory>
#include <string>
#include <vector>

#include "host_io.h"

namespace pb200 {

inline const char* pairwise_type_name(bool sparse) {
    return sparse ? "pecos::ann::PairwiseANN<pecos::ann::FeatVecSparseIPSimd<uint32_t, float>, pecos::csr_t>"
                  : "pecos::ann::PairwiseANN<pecos::ann::FeatVecDenseIPSimd<float>, pecos::drm_t>";
}

struct PairwiseHostModel {
    bool sparse = false;
    uint32_t num_input_keys = 0, num_label_keys = 0, feat_dim = 0;
    // Y_csc [N x L]: column l = rows row_idx[col_ptr[l] .. col_ptr[l+1]) with values y_val, in stored order
    const uint64_t* col_ptr = nullptr;
    const uint32_t* row_idx = nullptr;
    const float* y_val = nullptr;
    uint64_t nnz_y = 0;
    // X_trn [N x d]: dense row-major x_val, or csr (x_ptr, x_idx, x_val)
    const uint64_t* x_ptr = nullptr;
    const uint32_t* x_idx = nullptr;
    const float* x_val = nullptr;
    uint64_t nnz_x = 0;

    // owners: the mapped file (load) or deep copies (train)
    std::unique_ptr<MmapStoreReader> store;
    std::vector<uint64_t> own_col_ptr, own_x_ptr;
    std::vector<uint32_t> own_row_idx, own_x_idx;
    std::vector<float> own_y_val, own_x_val;

    uint32_t col_len(uint32_t label) const { return static_cast<uint32_t>(col_ptr[label + 1] - col_ptr[label]); }

    // Everything the device kernels rely on: offsets monotone and in range, every row id of Y a row of X.  The reference
    // reads out of bounds on such inputs; here they are refused before anything reaches the GPU.
    void validate() const {
        if (col_ptr[0] != 0 || col_ptr[num_label_keys] != nnz_y) throw std::runtime_error("pairwise_ann: Y_csc column offsets do not span its entries");
        for (uint32_t l = 0; l < num_label_keys; ++l)
            if (col_ptr[l + 1] < col_ptr[l]) throw std::runtime_error("pairwise_ann: Y_csc column offsets are not ascending");
        for (uint64_t e = 0; e < nnz_y; ++e)
            if (row_idx[e] >= num_input_keys) throw std::runtime_error("pairwise_ann: a row index of Y_csc is >= X_trn.rows");
        if (!sparse) {
            if (nnz_x != static_cast<uint64_t>(num_input_keys) * feat_dim) throw std::runtime_error("pairwise_ann: dense X_trn size mismatch");
            return;
        }
        if (x_ptr[0] != 0 || x_ptr[num_input_keys] != nnz_x) throw std::runtime_error("pairwise_ann: X_trn row offsets do not span its entries");
        for (uint32_t r = 0; r < num_input_keys; ++r)
            if (x_ptr[r + 1] < x_ptr[r]) throw std::runtime_error("pairwise_ann: X_trn row offsets are not ascending");
    }
};

// c_pairwise_ann_train_*: deep copies of X (dense or csr) and Y_csc (X rows = Y rows is required, as in the reference)
inline std::unique_ptr<PairwiseHostModel> pairwise_train(const HostMatrix& x, uint32_t y_rows, uint32_t y_cols, const uint64_t* y_ptr,
                                                         const uint32_t* y_idx, const float* y_val) {
    if (x.rows != y_rows) throw std::runtime_error("X_trn.rows != Y_csc.rows");
    const bool sparse = x.row_ptr != nullptr;
    auto m = std::make_unique<PairwiseHostModel>();
    m->sparse = sparse;
    m->num_input_keys = y_rows;
    m->num_label_keys = y_cols;
    m->feat_dim = x.cols;
    const uint64_t y0 = y_ptr[0];
    m->nnz_y = y_ptr[y_cols] - y0;
    m->own_col_ptr.resize(static_cast<size_t>(y_cols) + 1);
    for (uint32_t l = 0; l <= y_cols; ++l) m->own_col_ptr[l] = y_ptr[l] - y0;
    m->own_row_idx.assign(y_idx + y0, y_idx + y0 + m->nnz_y);
    m->own_y_val.assign(y_val + y0, y_val + y0 + m->nnz_y);
    if (sparse) {
        const uint64_t x0 = x.row_ptr[0];
        m->nnz_x = x.row_ptr[x.rows] - x0;
        m->own_x_ptr.resize(static_cast<size_t>(x.rows) + 1);
        for (uint32_t r = 0; r <= x.rows; ++r) m->own_x_ptr[r] = x.row_ptr[r] - x0;
        m->own_x_idx.assign(x.col_idx + x0, x.col_idx + x0 + m->nnz_x);
        m->own_x_val.assign(x.val + x0, x.val + x0 + m->nnz_x);
    } else {
        m->nnz_x = static_cast<uint64_t>(x.rows) * x.cols;
        m->own_x_val.assign(x.dense, x.dense + m->nnz_x);
    }
    m->col_ptr = m->own_col_ptr.data();
    m->row_idx = m->own_row_idx.data();
    m->y_val = m->own_y_val.data();
    m->x_ptr = sparse ? m->own_x_ptr.data() : nullptr;
    m->x_idx = sparse ? m->own_x_idx.data() : nullptr;
    m->x_val = m->own_x_val.data();
    m->validate();
    return m;
}

inline std::unique_ptr<PairwiseHostModel> load_pairwise_model(const std::string& model_dir, bool sparse, bool lazy_load) {
    JsonValue cfg = json_parse_file(model_dir + "/config.json");
    const std::string want = pairwise_type_name(sparse);
    const JsonValue* t = cfg.find("pairwise_ann_t");
    const std::string got = (t && t->kind == JsonValue::String) ? t->str : std::string("<missing>");
    if (got != want) throw std::invalid_argument("Inconsistent PairwiseANN_T: cur = " + want + " inp = " + got);
    const JsonValue* v = cfg.find("version");
    const std::string version = (v && v->kind == JsonValue::String) ? v->str : std::string("not found");
    if (version != "v1.0") throw std::runtime_error("Unable to load memory-mapped file with version = " + version);

    auto m = std::make_unique<PairwiseHostModel>();
    m->sparse = sparse;
    m->store = std::make_unique<MmapStoreReader>(model_dir + "/index.mmap_store", lazy_load);
    MmapStoreReader& s = *m->store;
    m->num_input_keys = s.get_one<uint32_t>();
    m->num_label_keys = s.get_one<uint32_t>();
    m->feat_dim = s.get_one<uint32_t>();
    const uint32_t y_rows = s.get_one<uint32_t>(), y_cols = s.get_one<uint32_t>();
    m->nnz_y = s.get_one<uint64_t>();
    m->col_ptr = s.get_multiple<uint64_t>(static_cast<uint64_t>(y_cols) + 1);
    m->row_idx = s.get_multiple<uint32_t>(m->nnz_y);
    m->y_val = s.get_multiple<float>(m->nnz_y);
    const uint32_t x_rows = s.get_one<uint32_t>(), x_cols = s.get_one<uint32_t>();
    m->nnz_x = s.get_one<uint64_t>();
    if (sparse) {
        m->x_ptr = s.get_multiple<uint64_t>(static_cast<uint64_t>(x_rows) + 1);
        m->x_idx = s.get_multiple<uint32_t>(m->nnz_x);
    }
    m->x_val = s.get_multiple<float>(m->nnz_x);
    if (y_rows != m->num_input_keys || y_cols != m->num_label_keys || x_rows != m->num_input_keys || x_cols != m->feat_dim)
        throw std::runtime_error("pairwise_ann index: matrix shapes disagree with N, L, d");
    m->validate();
    return m;
}

// PairwiseANN::save_config: nlohmann::json::dump(4) of the object below (keys sorted, no trailing newline)
inline std::string pairwise_config_json(const PairwiseHostModel& m) {
    return std::string("{\n    \"pairwise_ann_t\": \"") + pairwise_type_name(m.sparse) + "\",\n    \"train_params\": {\n" +
           "        \"feat_dim\": " + std::to_string(m.feat_dim) + ",\n        \"nnz_of_X\": " + std::to_string(m.nnz_x) +
           ",\n        \"nnz_of_Y\": " + std::to_string(m.nnz_y) + ",\n        \"num_input_keys\": " +
           std::to_string(m.num_input_keys) + ",\n        \"num_label_keys\": " + std::to_string(m.num_label_keys) +
           "\n    },\n    \"version\": \"v1.0\"\n}";
}

inline void save_pairwise_model(const PairwiseHostModel& m, const std::string& model_dir) {
    if (mkdir(model_dir.c_str(), 0777) == -1 && errno != EEXIST) throw std::runtime_error("Unable to create save folder at " + model_dir);
    {
        const std::string cfg = pairwise_config_json(m), path = model_dir + "/config.json";
        std::FILE* f = std::fopen(path.c_str(), "wb");
        if (!f) throw std::runtime_error("Unable to save config file to " + path);
        const bool ok = std::fwrite(cfg.data(), 1, cfg.size(), f) == cfg.size();
        if (std::fclose(f) != 0 || !ok) throw std::runtime_error("Unable to save config file to " + path);
    }
    MmapStoreWriter w(model_dir + "/index.mmap_store");
    w.put_one<uint32_t>(m.num_input_keys);
    w.put_one<uint32_t>(m.num_label_keys);
    w.put_one<uint32_t>(m.feat_dim);
    w.put_one<uint32_t>(m.num_input_keys);
    w.put_one<uint32_t>(m.num_label_keys);
    w.put_one<uint64_t>(m.nnz_y);
    w.put_multiple<uint64_t>(m.col_ptr, static_cast<uint64_t>(m.num_label_keys) + 1);
    w.put_multiple<uint32_t>(m.row_idx, m.nnz_y);
    w.put_multiple<float>(m.y_val, m.nnz_y);
    w.put_one<uint32_t>(m.num_input_keys);
    w.put_one<uint32_t>(m.feat_dim);
    w.put_one<uint64_t>(m.nnz_x);
    if (m.sparse) {
        w.put_multiple<uint64_t>(m.x_ptr, static_cast<uint64_t>(m.num_input_keys) + 1);
        w.put_multiple<uint32_t>(m.x_idx, m.nnz_x);
    }
    w.put_multiple<float>(m.x_val, m.nnz_x);
    w.close();
}

}  // namespace pb200
