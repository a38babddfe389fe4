// Host-side XR-Linear model ingest: on-disk model -> "chunked" layer layout that is uploaded to HBM.
//
// Reference behaviour restated here (nothing is copied; the layout is our own):
//   * model folder / metadata ............ pecos/core/xmc/inference.hpp:59-177, :2616-2655
//   * per-layer load (W.npz, C.npz) ....... pecos/core/xmc/inference.hpp:1568-1597
//   * contiguity check + rearrangement .... pecos/core/xmc/inference.hpp:652-668, :1745-1822, :1849-1883
//   * chunk construction .................. pecos/core/xmc/inference.hpp:557-650, :670-691
//   * compiled mmap layer ................. pecos/core/xmc/inference.hpp:413-455, :1886-1907; pecos/core/utils/matrix.hpp:386-407
//
// HBM layout of one layer (all arrays little-endian, element offsets not byte offsets):
//   chunks[n_chunks]   32-byte headers {col_begin, n_cols, nnz_rows, has_bias, meta_off u64, ent_off u64}
//   meta[]             per chunk: row_idx[R] padded with 0xFFFFFFFF to a multiple of 4 (16-byte aligned, so the
//                      kernel streams it with 128-bit loads), immediately followed by row_ptr[R+1] as u32 offsets
//                      RELATIVE to the chunk's first entry, again padded to a multiple of 4
//   entries[nnz]       {u32 col_offset, f32 val}, rows of a chunk stored consecutively in ascending feature order,
//                      inside a row ascending column (== the reference's chunk_entry_t order)
//   label_of_col[]     only when the tree was not contiguously ordered (pruned / permuted): rearranged col -> label id
#pragma once

#include <algorithm>
#include <cmath>
#include <thread>

#include "host_io.h"

namespace pb200 {

enum LayerTypeRequested { LT_CSC = 0, LT_HASH_CHUNKED = 1, LT_BINARY_SEARCH_CHUNKED = 2 };

enum PostProcKind { PP_NOOP = 0, PP_SIGMOID = 1, PP_LOG_SIGMOID = 2, PP_LP_HINGE = 3, PP_LOG_LP_HINGE = 4 };

struct PostProc {
    int kind = PP_NOOP;
    int p = 0;
};

// Name -> transform/combiner table, restating PostProcessor<T>::get (inference.hpp:192-240), including its
// fall-through for unknown names (identity transform, "keep x" combiner).
inline PostProc parse_post_processor(const std::string& name) {
    auto starts = [&](const char* s) { size_t n = strlen(s); return name.size() >= n && name.compare(0, n, s) == 0; };
    auto ends = [&](const char* s) { size_t n = strlen(s); return name.size() >= n && name.compare(name.size() - n, n, s) == 0; };
    PostProc pp;
    if (name == "noop") return pp;
    if (name == "sigmoid") { pp.kind = PP_SIGMOID; return pp; }
    if (name == "log-sigmoid") { pp.kind = PP_LOG_SIGMOID; return pp; }
    if (starts("log-l") && ends("-hinge")) {
        pp.kind = PP_LOG_LP_HINGE;
        pp.p = std::atoi(name.substr(5, name.size() - 5 - 6).c_str());
        return pp;
    }
    if (starts("l") && ends("-hinge")) {
        pp.kind = PP_LP_HINGE;
        pp.p = std::atoi(name.substr(1, name.size() - 1 - 6).c_str());
        return pp;
    }
    return pp;
}

struct CscHost {
    uint32_t rows = 0, cols = 0;
    std::vector<uint64_t> col_ptr;
    std::vector<uint32_t> row_idx;
    std::vector<float> val;
    uint64_t nnz() const { return col_ptr.empty() ? 0 : col_ptr[cols]; }
};

struct ChunkHeader {
    uint32_t col_begin;
    uint32_t n_cols;
    uint32_t nnz_rows;
    uint32_t has_bias;
    uint64_t meta_off;  // element offset into meta[] of this chunk's row_idx
    uint64_t ent_off;   // element offset into entries[] of this chunk's first entry
};
static_assert(sizeof(ChunkHeader) == 32, "chunk header must stay 32 bytes");

struct ChunkEntry {
    uint32_t col_offset;
    float val;
};
static_assert(sizeof(ChunkEntry) == 8, "chunk entry must stay 8 bytes");

inline uint64_t round_up4(uint64_t x) { return (x + 3) & ~uint64_t(3); }

struct uint2_host {
    uint32_t x, y;
};

struct ChunkedLayerHost {
    uint32_t w_rows = 0;     // W.rows (nr_features + 1 when bias > 0)
    uint32_t n_cols = 0;     // columns scored by this layer (after rearrangement: nnz(C))
    uint32_t out_cols = 0;   // column count reported for this layer's prediction matrix (perm.size() if rearranged)
    uint32_t n_chunks = 0;   // == C.cols == number of parent nodes
    uint32_t c_max = 0;      // widest chunk
    uint32_t r_max = 0;      // largest nnz_rows
    float bias = 1.0f;
    int only_topk = 10;
    std::string post_processor_name = "l3-hinge";
    PostProc post_processor;
    bool reordered = false;
    std::vector<ChunkHeader> chunks;
    std::vector<uint32_t> meta;
    std::vector<ChunkEntry> entries;
    std::vector<uint32_t> label_of_col;
    // Optional per-chunk feature map for query-driven lookups: fm_words = ceil(w_rows / 32) cells per chunk, cell w =
    // {bits: which of the features [32w, 32w+32) own a row in the chunk, prefix: number of chunk rows below 32w}.
    // slot(f) = prefix + popc(bits & ((1 << (f & 31)) - 1)) when bit f is set.  Built on request (build_feature_map).
    uint32_t fm_words = 0;
    std::vector<uint2_host> featmap;
};

struct XLinearHostModel {
    std::vector<ChunkedLayerHost> layers;
    int layer_type = LT_BINARY_SEARCH_CHUNKED;  // what the caller asked for; reported back verbatim
    bool is_mmap = false;
    uint32_t shard_rank = 0, shard_world = 1;   // leaf-layer index sharding (1 = whole model on this GPU)
    uint32_t leaf_chunk_begin = 0, leaf_chunk_end = 0;
    uint32_t depth() const { return static_cast<uint32_t>(layers.size()); }
    uint32_t nr_features() const {
        const auto& l = layers.back();
        return l.bias > 0.0f ? l.w_rows - 1 : l.w_rows;
    }
    // label_count() of the last layer: the chunked layouts report the columns of the (possibly rearranged / pruned) chunked
    // matrix, MLModel<csc_t> reports W.cols (inference.hpp:2367-2379) -- handles requested as CSC follow the latter
    uint32_t nr_labels() const { return layer_type == LT_CSC ? layers.back().out_cols : layers.back().n_cols; }
    uint32_t nr_codes() const { return layers.back().n_chunks; }
};

// ---------------------------------------------------------------------------------------------
// scipy npz -> CSC
// ---------------------------------------------------------------------------------------------
inline CscHost load_csc_npz(const std::string& path) {
    NpzFile npz(path);
    NpyView shape = npz.get("shape");
    NpyView indptr = npz.get("indptr");
    NpyView indices = npz.get("indices");
    NpyView data = npz.get("data");
    std::string fmt = npz.has("format") ? npz.get("format").as_text() : std::string("csc");
    if (shape.num_elements != 2) throw std::runtime_error("npz: bad shape member in " + path);
    uint64_t rows = shape.get_as<uint64_t>(0), cols = shape.get_as<uint64_t>(1);
    uint64_t nnz = data.num_elements;
    if (indices.num_elements != nnz) throw std::runtime_error("npz: indices/data size mismatch in " + path);

    CscHost m;
    m.rows = static_cast<uint32_t>(rows);
    m.cols = static_cast<uint32_t>(cols);
    if (fmt == "csc") {
        if (indptr.num_elements != cols + 1) throw std::runtime_error("npz: bad indptr length in " + path);
        m.col_ptr.resize(cols + 1);
        indptr.copy_to<uint64_t>(m.col_ptr.data());
        m.row_idx.resize(nnz);
        indices.copy_to<uint32_t>(m.row_idx.data());
        m.val.resize(nnz);
        data.copy_to<float>(m.val.data());
    } else if (fmt == "csr") {
        // transpose on the fly (the reference loader does the same through its csr->csc path)
        if (indptr.num_elements != rows + 1) throw std::runtime_error("npz: bad indptr length in " + path);
        std::vector<uint64_t> rp(rows + 1);
        indptr.copy_to<uint64_t>(rp.data());
        std::vector<uint32_t> ci(nnz);
        indices.copy_to<uint32_t>(ci.data());
        std::vector<float> v(nnz);
        data.copy_to<float>(v.data());
        m.col_ptr.assign(cols + 1, 0);
        for (uint64_t i = 0; i < nnz; ++i) m.col_ptr[ci[i] + 1]++;
        for (uint64_t c = 0; c < cols; ++c) m.col_ptr[c + 1] += m.col_ptr[c];
        m.row_idx.resize(nnz);
        m.val.resize(nnz);
        std::vector<uint64_t> fill(m.col_ptr.begin(), m.col_ptr.end() - 1);
        for (uint64_t r = 0; r < rows; ++r)
            for (uint64_t i = rp[r]; i < rp[r + 1]; ++i) {
                uint64_t dst = fill[ci[i]]++;
                m.row_idx[dst] = static_cast<uint32_t>(r);
                m.val[dst] = v[i];
            }
    } else {
        throw std::runtime_error("npz: unsupported sparse format '" + fmt + "' in " + path);
    }
    if (m.col_ptr[cols] != nnz) throw std::runtime_error("npz: indptr[-1] != nnz in " + path);
    return m;
}

inline CscHost csc_ones_column(uint32_t rows) {  // C of the root layer when C.npz is absent (inference.hpp:1580-1583)
    CscHost m;
    m.rows = rows; m.cols = 1;
    m.col_ptr = {0, rows};
    m.row_idx.resize(rows);
    m.val.assign(rows, 1.0f);
    for (uint32_t i = 0; i < rows; ++i) m.row_idx[i] = i;
    return m;
}

// ---------------------------------------------------------------------------------------------
// (W, C) -> chunked layer
// ---------------------------------------------------------------------------------------------
inline void build_chunked_layer(const CscHost& W, const CscHost& C, float bias, ChunkedLayerHost& L) {
    if (W.cols != C.rows) throw std::runtime_error("layer: W.cols != C.rows");
    const uint64_t c_nnz = C.nnz();
    // check_if_contiguously_ordered (inference.hpp:658-668)
    bool contiguous = (c_nnz >= C.rows);
    if (contiguous) {
        for (uint64_t i = 0; i < c_nnz; ++i) if (C.row_idx[i] != i) { contiguous = false; break; }
    }
    L.reordered = !contiguous;
    L.w_rows = W.rows;
    L.n_cols = static_cast<uint32_t>(c_nnz);   // rearranged column count (== W.cols when contiguous)
    L.out_cols = C.rows;                       // perm.size() (== W.cols when contiguous)
    L.n_chunks = C.cols;
    L.bias = bias;
    if (L.reordered) {
        // rearranged column j holds original column C.row_idx[j] (perm_inv, inference.hpp:1755-1759)
        L.label_of_col.assign(C.row_idx.begin(), C.row_idx.begin() + c_nnz);
        for (uint32_t lab : L.label_of_col)
            if (lab >= W.cols) throw std::runtime_error("layer: C row index out of range");
    }
    auto orig_col = [&](uint64_t j) -> uint32_t { return L.reordered ? L.label_of_col[j] : static_cast<uint32_t>(j); };

    // entry offsets per chunk are known up front: prefix of the rearranged column sizes
    L.chunks.assign(L.n_chunks, ChunkHeader{});
    std::vector<uint64_t> chunk_ent(L.n_chunks + 1, 0);
    for (uint32_t p = 0; p < L.n_chunks; ++p) {
        uint64_t cnt = 0;
        for (uint64_t j = C.col_ptr[p]; j < C.col_ptr[p + 1]; ++j) {
            uint32_t oc = orig_col(j);
            cnt += W.col_ptr[oc + 1] - W.col_ptr[oc];
        }
        chunk_ent[p + 1] = chunk_ent[p] + cnt;
    }
    L.entries.resize(chunk_ent[L.n_chunks]);

    const bool use_bias = bias > 0.0f;
    std::vector<std::vector<uint32_t>> chunk_rows(L.n_chunks), chunk_rptr(L.n_chunks);

    parallel_for_chunks(L.n_chunks, [&](uint64_t p) {
        struct Nz { uint64_t key; float val; };  // key = row << 32 | column offset; gather order is column-major so a
                                                 // stable sort on row alone == sort on (row, gather sequence)
        const uint64_t cb = C.col_ptr[p], ce = C.col_ptr[p + 1];
        const uint64_t n_ent = chunk_ent[p + 1] - chunk_ent[p];
        ChunkHeader& h = L.chunks[p];
        h.col_begin = static_cast<uint32_t>(cb);
        h.n_cols = static_cast<uint32_t>(ce - cb);
        h.ent_off = chunk_ent[p];
        h.nnz_rows = 0;
        h.has_bias = 0;
        if (n_ent == 0) { chunk_rptr[p].push_back(0); return; }
        if (n_ent >= (1ull << 32)) throw std::runtime_error("layer: a single chunk holds >= 2^32 entries");
        std::vector<Nz> nz(n_ent);
        uint64_t k = 0;
        for (uint64_t j = cb; j < ce; ++j) {
            uint32_t oc = orig_col(j);
            for (uint64_t i = W.col_ptr[oc]; i < W.col_ptr[oc + 1]; ++i) {
                nz[k].key = (static_cast<uint64_t>(W.row_idx[i]) << 32) | static_cast<uint64_t>(j - cb);
                nz[k].val = W.val[i];
                ++k;
            }
        }
        // stable on row only (duplicates of (row, col) keep their column-major order, like the reference)
        std::stable_sort(nz.begin(), nz.end(), [](const Nz& a, const Nz& b) { return (a.key >> 32) < (b.key >> 32); });
        auto& rows = chunk_rows[p];
        auto& rptr = chunk_rptr[p];
        ChunkEntry* out = L.entries.data() + h.ent_off;
        uint32_t last_row = 0xFFFFFFFFu;
        bool first = true;
        for (uint64_t i = 0; i < n_ent; ++i) {
            uint32_t r = static_cast<uint32_t>(nz[i].key >> 32);
            uint32_t co = static_cast<uint32_t>(nz[i].key & 0xFFFFFFFFu);
            if (first || r != last_row) {
                rows.push_back(r);
                rptr.push_back(static_cast<uint32_t>(i));
                last_row = r;
                first = false;
            }
            out[i].col_offset = co;
            out[i].val = nz[i].val;
        }
        rptr.push_back(static_cast<uint32_t>(n_ent));
        h.nnz_rows = static_cast<uint32_t>(rows.size());
        // check_bias_explicit (inference.hpp:500-502) gated by bias > 0 (inference.hpp:679-690)
        h.has_bias = (use_bias && rows.back() == W.rows - 1) ? 1u : 0u;
    });

    uint64_t meta_total = 0;
    L.c_max = 0; L.r_max = 0;
    for (uint32_t p = 0; p < L.n_chunks; ++p) {
        ChunkHeader& h = L.chunks[p];
        h.meta_off = meta_total;
        meta_total += round_up4(h.nnz_rows) + round_up4(static_cast<uint64_t>(h.nnz_rows) + 1);
        L.c_max = std::max(L.c_max, h.n_cols);
        L.r_max = std::max(L.r_max, h.nnz_rows);
    }
    L.meta.assign(meta_total, 0xFFFFFFFFu);
    parallel_for_chunks(L.n_chunks, [&](uint64_t p) {
        const ChunkHeader& h = L.chunks[p];
        uint32_t* m = L.meta.data() + h.meta_off;
        std::copy(chunk_rows[p].begin(), chunk_rows[p].end(), m);
        uint32_t* rp = m + round_up4(h.nnz_rows);
        std::copy(chunk_rptr[p].begin(), chunk_rptr[p].end(), rp);
    });
}

// ---------------------------------------------------------------------------------------------
// index sharding of the leaf layer (SURVEY.md 8e): rank r of `world` keeps the weights of a contiguous range of leaf
// chunks, balanced by entry bytes; every other chunk keeps only its header (column range => candidate positions stay
// global) and is flagged absent (bit 1 of has_bias).  Upper layers are replicated.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kChunkAbsent = 2u;

inline void shard_ranges_by_weight(const std::vector<uint64_t>& weight, uint32_t world, std::vector<uint32_t>& begin) {
    // begin[r] .. begin[r+1] = chunks of rank r; greedy split at the prefix-sum quantiles
    const uint32_t n = static_cast<uint32_t>(weight.size());
    uint64_t total = 0;
    for (uint64_t w : weight) total += w + 1;
    begin.assign(world + 1, n);
    begin[0] = 0;
    uint64_t run = 0;
    uint32_t r = 1;
    for (uint32_t i = 0; i < n && r < world; ++i) {
        run += weight[i] + 1;
        while (r < world && run * world >= static_cast<uint64_t>(r) * total) begin[r++] = i + 1;
    }
    for (; r < world; ++r) begin[r] = n;
}

inline void apply_leaf_shard(ChunkedLayerHost& L, uint32_t rank, uint32_t world, uint32_t& c0, uint32_t& c1) {
    if (world <= 1) { c0 = 0; c1 = L.n_chunks; return; }
    if (rank >= world) throw std::runtime_error("leaf shard: rank >= world");
    std::vector<uint64_t> weight(L.n_chunks);
    for (uint32_t p = 0; p < L.n_chunks; ++p) {
        const ChunkHeader& h = L.chunks[p];
        const uint32_t* rp = L.meta.data() + h.meta_off + round_up4(h.nnz_rows);
        weight[p] = static_cast<uint64_t>(rp[h.nnz_rows]) * 8 + static_cast<uint64_t>(h.nnz_rows) * 8;
    }
    std::vector<uint32_t> begin;
    shard_ranges_by_weight(weight, world, begin);
    c0 = begin[rank];
    c1 = begin[rank + 1];
    std::vector<uint32_t> meta;
    std::vector<ChunkEntry> entries;
    for (uint32_t p = 0; p < L.n_chunks; ++p) {
        ChunkHeader& h = L.chunks[p];
        if (p >= c0 && p < c1) {
            const uint64_t m_len = round_up4(h.nnz_rows) + round_up4(static_cast<uint64_t>(h.nnz_rows) + 1);
            const uint32_t* src_m = L.meta.data() + h.meta_off;
            const uint32_t n_ent = src_m[round_up4(h.nnz_rows) + h.nnz_rows];
            const ChunkEntry* src_e = L.entries.data() + h.ent_off;
            h.meta_off = meta.size();
            h.ent_off = entries.size();
            meta.insert(meta.end(), src_m, src_m + m_len);
            entries.insert(entries.end(), src_e, src_e + n_ent);
        } else {
            h.nnz_rows = 0;
            h.has_bias = kChunkAbsent;
            h.meta_off = 0;
            h.ent_off = 0;
        }
    }
    if (meta.empty()) meta.assign(4, 0u);  // keep device pointers valid on ranks that own nothing
    L.meta.swap(meta);
    L.entries.swap(entries);
}

// The two upper layers as ONE one-chunk layer: W = [W0 | W1] with layer 1's columns in its (contiguous) column order, one
// shared bias row.  A column's raw score is the sum over its own entries only, so scoring this layer gives both layers'
// raw scores bit for bit.  Needs the host arrays of both layers, neither rearranged, the same feature space and the same
// bias.
inline void build_prefix_layer(const ChunkedLayerHost& L0, const ChunkedLayerHost& L1, ChunkedLayerHost& M) {
    if (L0.reordered || L1.reordered || L0.w_rows != L1.w_rows) throw std::runtime_error("prefix layer: layers do not merge");
    CscHost W;
    W.rows = L0.w_rows;
    W.cols = L0.n_cols + L1.n_cols;
    W.col_ptr.assign(static_cast<size_t>(W.cols) + 1, 0);
    // chunk c of layer l holds merged columns [first + col_begin, first + col_begin + n_cols); its rows ascend, so appending
    // row by row keeps every column's entries in row order
    auto for_each_entry = [&](auto&& fn) {
        uint32_t first = 0;
        for (const ChunkedLayerHost* L : {&L0, &L1}) {
            for (const ChunkHeader& h : L->chunks) {
                const uint32_t* rows = L->meta.data() + h.meta_off;
                const uint32_t* rp = rows + round_up4(h.nnz_rows);
                const ChunkEntry* en = L->entries.data() + h.ent_off;
                for (uint32_t r = 0; r < h.nnz_rows; ++r)
                    for (uint32_t i = rp[r]; i < rp[r + 1]; ++i) fn(first + h.col_begin + en[i].col_offset, rows[r], en[i].val);
            }
            first += L->n_cols;
        }
    };
    for_each_entry([&](uint32_t col, uint32_t, float) { ++W.col_ptr[col + 1]; });
    for (uint32_t c = 0; c < W.cols; ++c) W.col_ptr[c + 1] += W.col_ptr[c];
    W.row_idx.resize(W.nnz());
    W.val.resize(W.nnz());
    std::vector<uint64_t> fill(W.col_ptr.begin(), W.col_ptr.end() - 1);
    for_each_entry([&](uint32_t col, uint32_t row, float v) {
        W.row_idx[fill[col]] = row;
        W.val[fill[col]++] = v;
    });
    build_chunked_layer(W, csc_ones_column(W.cols), L0.bias, M);
}

// Bytes the feature map of a layer would occupy.
inline uint64_t feature_map_bytes(const ChunkedLayerHost& L) {
    return static_cast<uint64_t>(L.n_chunks) * ((static_cast<uint64_t>(L.w_rows) + 31) / 32) * 8;
}

// Builds the per-chunk {bits, prefix} cells from the chunk row lists (must run before meta[] is released).
inline void build_feature_map(ChunkedLayerHost& L) {
    L.fm_words = static_cast<uint32_t>((static_cast<uint64_t>(L.w_rows) + 31) / 32);
    L.featmap.assign(static_cast<uint64_t>(L.n_chunks) * L.fm_words, uint2_host{0u, 0u});
    parallel_for_chunks(L.n_chunks, [&](uint64_t p) {
        const ChunkHeader& h = L.chunks[p];
        const uint32_t* rows = L.meta.data() + h.meta_off;
        uint2_host* cells = L.featmap.data() + p * L.fm_words;
        for (uint32_t r = 0; r < h.nnz_rows; ++r) cells[rows[r] >> 5].x |= 1u << (rows[r] & 31u);
        uint32_t run = 0;
        for (uint32_t w = 0; w < L.fm_words; ++w) {
            cells[w].y = run;
            run += static_cast<uint32_t>(__builtin_popcount(cells[w].x));
        }
    });
}

// ---------------------------------------------------------------------------------------------
// layer / model loaders
// ---------------------------------------------------------------------------------------------
struct LayerMeta {
    float bias = 1.0f;
    int only_topk = 10;
    std::string post_processor = "l3-hinge";
    bool is_mmap = false;
};

inline LayerMeta load_layer_meta(const std::string& path) {
    // restates MLModelMetadata(const std::string&) (inference.hpp:120-157)
    JsonValue j = json_parse_file(path);
    const JsonValue* model = j.find("model");
    std::string model_type = (model && model->kind == JsonValue::String) ? model->str : "None";
    if (model_type != "MLModel") throw std::runtime_error(model_type + " loading is not implemented");
    if (!j.contains("bias")) throw std::runtime_error("model corrupted, does not contain bias");
    if (!j.contains("pred_kwargs")) throw std::runtime_error("model corrupted, does not contain pred_kwargs");
    const JsonValue& pk = j.at("pred_kwargs");
    if (!pk.contains("only_topk")) throw std::runtime_error("model corrupted, does not contain only_topk in pred_kwargs");
    if (!pk.contains("post_processor")) throw std::runtime_error("model corrupted, does not contain post_processor in pred_kwargs");
    LayerMeta m;
    m.bias = static_cast<float>(j.at("bias").as_number());
    m.only_topk = static_cast<int>(pk.at("only_topk").as_number());
    m.post_processor = pk.at("post_processor").as_string();
    const JsonValue* mm = j.find("is_mmap");
    m.is_mmap = mm ? mm->as_bool() : false;
    return m;
}

inline void apply_meta(const LayerMeta& m, ChunkedLayerHost& L) {
    L.bias = m.bias;
    L.only_topk = m.only_topk;
    L.post_processor_name = m.post_processor;
    L.post_processor = parse_post_processor(m.post_processor);
}

inline void load_npz_layer(const std::string& folder, uint32_t depth, ChunkedLayerHost& L) {
    LayerMeta meta = load_layer_meta(folder + "/param.json");
    CscHost W = load_csc_npz(folder + "/W.npz");
    CscHost C;
    const std::string c_path = folder + "/C.npz";
    if (depth == 0 && !file_exists(c_path)) C = csc_ones_column(W.cols);
    else C = load_csc_npz(c_path);
    build_chunked_layer(W, C, meta.bias, L);
    apply_meta(meta, L);
}

// One-layer model from in-memory CSC matrices (c_xlinear_single_layer_predict_*: the python prediction chain hands W and
// C of a layer to the native side on every call, pecos/core/libpecos.cpp:201-235).  The arrays are copied.
struct CscRaw {
    uint32_t rows, cols;
    const uint64_t* col_ptr;
    const uint32_t* row_idx;
    const float* val;
};

inline CscHost copy_csc(const CscRaw& A) {
    if (A.cols && !A.col_ptr) throw std::runtime_error("single layer: null col_ptr");
    CscHost H;
    H.rows = A.rows;
    H.cols = A.cols;
    H.col_ptr.assign(A.col_ptr, A.col_ptr + static_cast<size_t>(A.cols) + 1);
    const uint64_t nnz = H.col_ptr[A.cols];
    if (H.col_ptr[0] != 0) throw std::runtime_error("single layer: col_ptr[0] != 0");
    for (uint32_t c = 0; c < A.cols; ++c)
        if (H.col_ptr[c] > H.col_ptr[c + 1]) throw std::runtime_error("single layer: col_ptr is not monotone");
    H.row_idx.assign(A.row_idx, A.row_idx + nnz);
    H.val.assign(A.val, A.val + nnz);
    for (uint64_t i = 0; i < nnz; ++i)
        if (H.row_idx[i] >= A.rows) throw std::runtime_error("single layer: row index out of range");
    return H;
}

inline std::unique_ptr<XLinearHostModel> make_single_layer_model(const CscRaw& W, const CscRaw& C, float bias) {
    auto m = std::make_unique<XLinearHostModel>();
    m->layer_type = LT_CSC;  // what the reference instantiates here: MLModel<csc_t> (same results, see DESIGN.md 3.1)
    m->layers.resize(1);
    const CscHost Wh = copy_csc(W);
    const CscHost Ch = copy_csc(C);
    build_chunked_layer(Wh, Ch, bias, m->layers[0]);
    LayerMeta meta;
    meta.bias = bias;
    apply_meta(meta, m->layers[0]);
    m->leaf_chunk_begin = 0;
    m->leaf_chunk_end = m->layers[0].n_chunks;
    return m;
}

// csc_t::load_from_mmap_store (pecos/core/utils/matrix.hpp:398-407): [rows u32][cols u32][nnz u64][col_ptr][row_idx][val]
inline CscHost load_csc_mmap(const std::string& path, bool lazy_load) {
    MmapStoreReader s(path, lazy_load);
    CscHost m;
    m.rows = s.get_one<uint32_t>();
    m.cols = s.get_one<uint32_t>();
    const uint64_t nnz = s.get_one<uint64_t>();
    const uint64_t* cp = s.get_multiple<uint64_t>(static_cast<uint64_t>(m.cols) + 1);
    const uint32_t* ri = s.get_multiple<uint32_t>(nnz);
    const float* v = s.get_multiple<float>(nnz);
    if (cp[m.cols] != nnz) throw std::runtime_error("mmap csc: col_ptr[-1] != nnz in " + path);
    m.col_ptr.assign(cp, cp + m.cols + 1);
    m.row_idx.assign(ri, ri + nnz);
    m.val.assign(v, v + nnz);
    return m;
}

// c_mlmodel_load_mmap_model (pecos/core/libpecos.cpp:37-40): ONE layer saved by MLModel<csc_t>::save_mmap
// (inference.hpp:2274-2289: param.json with is_mmap = true, W.mmap_store and C.mmap_store in csc_t's mmap format).
inline std::unique_ptr<XLinearHostModel> load_mlmodel_mmap(const std::string& folder, bool lazy_load) {
    LayerMeta meta = load_layer_meta(folder + "/param.json");
    if (!meta.is_mmap) throw std::runtime_error("This folder contains npz model. Cannot load in mmap format.");
    auto m = std::make_unique<XLinearHostModel>();
    m->layer_type = LT_CSC;
    m->is_mmap = true;
    m->layers.resize(1);
    const CscHost W = load_csc_mmap(folder + "/W.mmap_store", lazy_load);
    const CscHost C = load_csc_mmap(folder + "/C.mmap_store", lazy_load);
    build_chunked_layer(W, C, meta.bias, m->layers[0]);
    apply_meta(meta, m->layers[0]);
    m->leaf_chunk_begin = 0;
    m->leaf_chunk_end = m->layers[0].n_chunks;
    return m;
}

// Compiled layer: W.mmap_store already holds the reference's chunked arrays; we only re-pack them.
inline void load_mmap_layer(const std::string& folder, bool lazy_load, ChunkedLayerHost& L) {
    LayerMeta meta = load_layer_meta(folder + "/param.json");
    struct RefChunk { uint32_t col_begin, col_end, nnz_rows, has_bias; uint64_t p0, p1; };  // 32-byte on-disk struct
    static_assert(sizeof(RefChunk) == 32, "on-disk chunk struct is 32 bytes");
    {
        MmapStoreReader ws(folder + "/W.mmap_store", lazy_load);
        uint32_t chunk_count = ws.get_one<uint32_t>();
        uint32_t rows = ws.get_one<uint32_t>();
        uint32_t cols = ws.get_one<uint32_t>();
        uint64_t n_chunks_v, n_ridx, n_rptr, n_ent;
        const RefChunk* rc = ws.get_vector<RefChunk>(&n_chunks_v);
        const uint32_t* ridx = ws.get_vector<uint32_t>(&n_ridx);
        const uint64_t* rptr = ws.get_vector<uint64_t>(&n_rptr);
        const ChunkEntry* ent = ws.get_vector<ChunkEntry>(&n_ent);
        if (n_chunks_v != chunk_count) throw std::runtime_error("mmap layer: chunk count mismatch");
        L.w_rows = rows;
        L.n_cols = cols;
        L.out_cols = cols;
        L.n_chunks = chunk_count;
        L.chunks.assign(chunk_count, ChunkHeader{});
        L.entries.assign(ent, ent + n_ent);
        uint64_t meta_total = 0, ri = 0, rp = 0;
        std::vector<uint64_t> src_ridx(chunk_count), src_rptr(chunk_count);
        L.c_max = 0; L.r_max = 0;
        for (uint32_t p = 0; p < chunk_count; ++p) {
            ChunkHeader& h = L.chunks[p];
            h.col_begin = rc[p].col_begin;
            h.n_cols = rc[p].col_end - rc[p].col_begin;
            h.nnz_rows = rc[p].nnz_rows;
            h.has_bias = rc[p].has_bias ? 1u : 0u;
            h.meta_off = meta_total;
            meta_total += round_up4(h.nnz_rows) + round_up4(static_cast<uint64_t>(h.nnz_rows) + 1);
            src_ridx[p] = ri; src_rptr[p] = rp;
            if (h.nnz_rows) { ri += h.nnz_rows; rp += h.nnz_rows + 1; }
            L.c_max = std::max(L.c_max, h.n_cols);
            L.r_max = std::max(L.r_max, h.nnz_rows);
        }
        if (ri != n_ridx || rp != n_rptr) throw std::runtime_error("mmap layer: row index arrays have unexpected size");
        L.meta.assign(meta_total, 0xFFFFFFFFu);
        uint64_t ent_cursor = 0;
        for (uint32_t p = 0; p < chunk_count; ++p) {
            ChunkHeader& h = L.chunks[p];
            uint32_t* m = L.meta.data() + h.meta_off;
            uint32_t* out_rp = m + round_up4(h.nnz_rows);
            if (h.nnz_rows == 0) { h.ent_off = ent_cursor; out_rp[0] = 0; continue; }
            const uint64_t* in_rp = rptr + src_rptr[p];
            h.ent_off = in_rp[0];
            for (uint32_t r = 0; r < h.nnz_rows; ++r) m[r] = ridx[src_ridx[p] + r];
            for (uint32_t r = 0; r <= h.nnz_rows; ++r) {
                uint64_t rel = in_rp[r] - in_rp[0];
                if (rel >= (1ull << 32)) throw std::runtime_error("mmap layer: a single chunk holds >= 2^32 entries");
                out_rp[r] = static_cast<uint32_t>(rel);
            }
            ent_cursor = in_rp[h.nnz_rows];
        }
    }
    {
        // C.mmap_store is only needed for its column count sanity check; chunk headers already encode the tree.
        MmapStoreReader cs(folder + "/C.mmap_store", lazy_load);
        uint32_t c_rows = cs.get_one<uint32_t>();
        uint32_t c_cols = cs.get_one<uint32_t>();
        if (c_cols != L.n_chunks) throw std::runtime_error("mmap layer: C.cols != chunk count");
        if (c_rows != L.n_cols) throw std::runtime_error("mmap layer: C.rows != W.cols");
    }
    const std::string perm_path = folder + "/perm.mmap_store";
    if (file_exists(perm_path)) {
        MmapStoreReader ps(perm_path, lazy_load);
        uint64_t n_perm, n_inv;
        (void)ps.get_vector<uint32_t>(&n_perm);
        const uint32_t* inv = ps.get_vector<uint32_t>(&n_inv);
        L.reordered = true;
        L.label_of_col.assign(inv, inv + n_inv);
        L.out_cols = static_cast<uint32_t>(n_perm);
    } else {
        L.reordered = false;
    }
    apply_meta(meta, L);
}

// c_xlinear_compile_mmap_model (pecos/core/libpecos.cpp:133-138; HierarchicalMLModel::save_mmap inference.hpp:2575-2595, layer
// :1907-1916, chunked matrix :413-423, csc_t matrix.hpp:386-396, rearrangement :1716-1728): writes a model in the reference's
// mmap format from our host layout -- the same arrays, u64 row pointers global to the layer's entry array.  Needs the host
// arrays, i.e. a model that has not been handed to an engine yet.
inline void write_json_text(const std::string& path, const std::string& text) {
    std::FILE* f = std::fopen(path.c_str(), "wb");
    if (!f) throw std::runtime_error("could not open " + path);
    std::fwrite(text.data(), 1, text.size(), f);
    std::fclose(f);
}

inline void write_xlinear_mmap_model(const XLinearHostModel& m, const std::string& folder) {
    if (system(("mkdir -p '" + folder + "'").c_str()) != 0) throw std::runtime_error("Cannot create folder: " + folder);
    write_json_text(folder + "/param.json",
                    "{\n\"model\": \"HierarchicalMLModel\",\n\"depth\": " + std::to_string(m.depth()) + ",\n\"is_mmap\": true\n}\n");
    for (uint32_t d = 0; d < m.depth(); ++d) {
        const ChunkedLayerHost& L = m.layers[d];
        if (L.meta.empty() && !L.chunks.empty() && L.n_cols > 0 && L.entries.empty())
            throw std::runtime_error("write_xlinear_mmap_model: the host arrays of this model were already released");
        const std::string lf = folder + "/" + std::to_string(d) + ".model";
        if (system(("mkdir -p '" + lf + "'").c_str()) != 0) throw std::runtime_error("Cannot create folder: " + lf);
        char bias_txt[64];
        std::snprintf(bias_txt, sizeof(bias_txt), "%.9g", static_cast<double>(L.bias));
        write_json_text(lf + "/param.json",
                        std::string("{\n\"model\": \"MLModel\",\n\"bias\": ") + bias_txt + ",\n\"pred_kwargs\": {\n\t\"only_topk\": " +
                            std::to_string(L.only_topk) + ",\n\t\"post_processor\": \"" + L.post_processor_name +
                            "\"\n\t},\n\"is_mmap\": true\n}\n");
        {   // W.mmap_store
            struct RefChunk { uint32_t col_begin, col_end, nnz_rows, has_bias; uint64_t p0, p1; };
            std::vector<RefChunk> rc(L.n_chunks);
            std::vector<uint32_t> ridx;
            std::vector<uint64_t> rptr;
            uint64_t ent_total = 0;
            for (uint32_t p = 0; p < L.n_chunks; ++p) {
                const ChunkHeader& h = L.chunks[p];
                if (h.has_bias & kChunkAbsent) throw std::runtime_error("write_xlinear_mmap_model: index-sharded models cannot be written");
                rc[p] = RefChunk{h.col_begin, h.col_begin + h.n_cols, h.nnz_rows, (h.has_bias & 1u) ? 1u : 0u, 0, 0};
                if (h.nnz_rows == 0) continue;
                const uint32_t* mi = L.meta.data() + h.meta_off;
                const uint32_t* rp = mi + round_up4(h.nnz_rows);
                ridx.insert(ridx.end(), mi, mi + h.nnz_rows);
                for (uint32_t r = 0; r <= h.nnz_rows; ++r) rptr.push_back(h.ent_off + rp[r]);
                ent_total = std::max<uint64_t>(ent_total, h.ent_off + rp[h.nnz_rows]);
            }
            MmapStoreWriter w(lf + "/W.mmap_store");
            w.put_one<uint32_t>(L.n_chunks);
            w.put_one<uint32_t>(L.w_rows);
            w.put_one<uint32_t>(L.n_cols);
            w.put_vector<RefChunk>(rc.data(), rc.size());
            w.put_vector<uint32_t>(ridx.data(), ridx.size());
            w.put_vector<uint64_t>(rptr.data(), rptr.size());
            w.put_vector<ChunkEntry>(L.entries.data(), L.entries.size());
            w.close();
        }
        {   // C.mmap_store: the (rearranged) code matrix -- column p holds the contiguous rows [col_begin, col_end) of chunk p
            std::vector<uint64_t> col_ptr(static_cast<size_t>(L.n_chunks) + 1, 0);
            for (uint32_t p = 0; p < L.n_chunks; ++p) col_ptr[p + 1] = col_ptr[p] + L.chunks[p].n_cols;
            const uint64_t nnz = col_ptr[L.n_chunks];
            std::vector<uint32_t> row_idx(nnz);
            for (uint32_t p = 0; p < L.n_chunks; ++p)
                for (uint32_t j = 0; j < L.chunks[p].n_cols; ++j) row_idx[col_ptr[p] + j] = L.chunks[p].col_begin + j;
            std::vector<float> val(nnz, 1.0f);
            MmapStoreWriter w(lf + "/C.mmap_store");
            w.put_one<uint32_t>(L.n_cols);
            w.put_one<uint32_t>(L.n_chunks);
            w.put_one<uint64_t>(nnz);
            w.put_multiple<uint64_t>(col_ptr.data(), col_ptr.size());
            w.put_multiple<uint32_t>(row_idx.data(), nnz);
            w.put_multiple<float>(val.data(), nnz);
            w.close();
        }
        if (L.reordered) {  // perm[label] = rearranged position (nnz(C) for labels without a parent), perm_inv = its inverse
            std::vector<uint32_t> perm(L.out_cols, static_cast<uint32_t>(L.label_of_col.size()));
            for (uint32_t i = 0; i < L.label_of_col.size(); ++i)
                if (L.label_of_col[i] < L.out_cols) perm[L.label_of_col[i]] = i;
            MmapStoreWriter w(lf + "/perm.mmap_store");
            w.put_vector<uint32_t>(perm.data(), perm.size());
            w.put_vector<uint32_t>(L.label_of_col.data(), L.label_of_col.size());
            w.close();
        }
    }
}

// c_mlmodel_compile_mmap_model (pecos/core/libpecos.cpp:32-36; MLModel<csc_t>::save_mmap inference.hpp:2274-2289, LayerData<csc_t>
// :1676-1680, csc_t::save_to_mmap_store matrix.hpp:386-396): ONE npz layer folder (param.json + W.npz + C.npz; the root layer may
// lack C.npz = one parent holding every label, inference.hpp:1580-1583) -> param.json (is_mmap = true) + W.mmap_store + C.mmap_store,
// both in csc_t's layout [rows u32][cols u32][nnz u64][col_ptr u64 x (cols + 1)][row_idx u32 x nnz][val f32 x nnz].  Host-only.
inline void write_csc_mmap(const CscHost& A, const std::string& path) {
    MmapStoreWriter w(path);
    w.put_one<uint32_t>(A.rows);
    w.put_one<uint32_t>(A.cols);
    w.put_one<uint64_t>(A.nnz());
    w.put_multiple<uint64_t>(A.col_ptr.data(), static_cast<uint64_t>(A.cols) + 1);
    w.put_multiple<uint32_t>(A.row_idx.data(), A.nnz());
    w.put_multiple<float>(A.val.data(), A.nnz());
    w.close();
}

inline void compile_mlmodel_mmap(const std::string& npz_folder, const std::string& mmap_folder) {
    const LayerMeta meta = load_layer_meta(npz_folder + "/param.json");
    if (meta.is_mmap) throw std::runtime_error("This folder contains mmap model. Cannot load in npz format.");
    const CscHost W = load_csc_npz(npz_folder + "/W.npz");
    const std::string c_path = npz_folder + "/C.npz";
    const CscHost C = file_exists(c_path) ? load_csc_npz(c_path) : csc_ones_column(W.cols);
    if (system(("mkdir -p '" + mmap_folder + "'").c_str()) != 0) throw std::runtime_error("Cannot create folder: " + mmap_folder);
    char bias_txt[64];
    std::snprintf(bias_txt, sizeof(bias_txt), "%.9g", static_cast<double>(meta.bias));
    write_json_text(mmap_folder + "/param.json",
                    std::string("{\n\"model\": \"MLModel\",\n\"bias\": ") + bias_txt + ",\n\"pred_kwargs\": {\n\t\"only_topk\": " +
                        std::to_string(meta.only_topk) + ",\n\t\"post_processor\": \"" + meta.post_processor +
                        "\"\n\t},\n\"is_mmap\": true\n}\n");
    write_csc_mmap(W, mmap_folder + "/W.mmap_store");
    write_csc_mmap(C, mmap_folder + "/C.mmap_store");
}

struct HierMeta { int depth = 0; bool is_mmap = false; };

inline HierMeta load_hier_meta(const std::string& path) {
    // restates HierarchicalMLModelMetadata (inference.hpp:65-84)
    JsonValue j = json_parse_file(path);
    const JsonValue* model = j.find("model");
    std::string model_type = (model && model->kind == JsonValue::String) ? model->str : "None";
    if (model_type != "HierarchicalMLModel") throw std::runtime_error(model_type + " loading is not implemented");
    HierMeta m;
    const JsonValue* d = j.find("depth");
    m.depth = d ? static_cast<int>(d->as_number()) : -1;
    if (m.depth <= 0) throw std::runtime_error("model corrupted, depth is 0 or negative");
    const JsonValue* mm = j.find("is_mmap");
    m.is_mmap = mm ? mm->as_bool() : false;
    return m;
}

inline std::unique_ptr<XLinearHostModel> load_xlinear_npz_model(const std::string& folder, int layer_type,
                                                                uint32_t shard_rank = 0, uint32_t shard_world = 1) {
    HierMeta hm = load_hier_meta(folder + "/param.json");
    if (hm.is_mmap) throw std::runtime_error("This folder contains mmap model. Cannot load in npz format.");
    auto model = std::make_unique<XLinearHostModel>();
    model->layer_type = (layer_type == LT_CSC || layer_type == LT_HASH_CHUNKED) ? layer_type : LT_BINARY_SEARCH_CHUNKED;
    model->is_mmap = false;
    model->layers.resize(hm.depth);
    for (int d = 0; d < hm.depth; ++d)
        load_npz_layer(folder + "/" + std::to_string(d) + ".model", static_cast<uint32_t>(d), model->layers[d]);
    model->shard_rank = shard_rank;
    model->shard_world = std::max<uint32_t>(shard_world, 1u);
    apply_leaf_shard(model->layers.back(), shard_rank, model->shard_world, model->leaf_chunk_begin, model->leaf_chunk_end);
    return model;
}

inline std::unique_ptr<XLinearHostModel> load_xlinear_mmap_model(const std::string& folder, bool lazy_load,
                                                                 uint32_t shard_rank = 0, uint32_t shard_world = 1) {
    HierMeta hm = load_hier_meta(folder + "/param.json");
    if (!hm.is_mmap) throw std::runtime_error("This folder contains npz model. Cannot load in mmap format.");
    auto model = std::make_unique<XLinearHostModel>();
    model->layer_type = LT_BINARY_SEARCH_CHUNKED;
    model->is_mmap = true;
    model->layers.resize(hm.depth);
    for (int d = 0; d < hm.depth; ++d)
        load_mmap_layer(folder + "/" + std::to_string(d) + ".model", lazy_load, model->layers[d]);
    model->shard_rank = shard_rank;
    model->shard_world = std::max<uint32_t>(shard_world, 1u);
    apply_leaf_shard(model->layers.back(), shard_rank, model->shard_world, model->leaf_chunk_begin, model->leaf_chunk_end);
    return model;
}

}  // namespace pb200
