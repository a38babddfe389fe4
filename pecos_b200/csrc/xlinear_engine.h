// XR-Linear beam-search engine on one H100: device-resident model + the two kernels per tree layer.
//
// Replaces (reference, CPU/OpenMP):
//   HierarchicalMLModel::predict ........ pecos/core/xmc/inference.hpp:2446-2488
//   MLModel::predict_internal ........... pecos/core/xmc/inference.hpp:2029-2080
//     prolongate_predictions ............ :1155-1219   (implicit here: beam slot j -> chunk j, no materialised pattern)
//     w_ops::compute_sparse_predictions . :925-1007    -> xl_chunk_scores_kernel
//       chunk_ops<csr|drm, bin_search> .. :769-839
//     transform / combine / sorted_csr .. :1360-1384, :1223-1298 -> xl_topk_kernel
//     reorder_prediction ................ :1919-1923   (label_of_col lookup in xl_topk_kernel)
#pragma once

#include <functional>
#include <memory>
#include <string>
#include <vector>

#include "cuda_util.h"
#include "xlinear_host.h"

namespace pb200 {

struct LayerDev {
    const ChunkHeader* chunks;
    const uint32_t* meta;
    const uint32_t* rowext;        // same indexing as meta: chunk region [meta_off, meta_off + 2R) = {begin, end} per row
    const uint2* entries;
    const uint32_t* label_of_col;  // nullptr when the layer is contiguously ordered
    const uint2* featmap;          // per-chunk {bits, prefix} cells for query-driven lookups; nullptr = stream row lists
    uint32_t fm_words;
    uint32_t n_cols;
    uint32_t n_chunks;
    uint32_t c_max;
    uint32_t w_rows;
    float bias;
};

// Chunk-major score kernel (xlinear_cm_kernel.cuh)
struct CmShape {  // load-time, per layer: geometry of the chunk images
    bool ok = false;
    bool direct = false;
    uint32_t words = 0;      // direct: w_rows + 1 (u16 row starts); else fm_words (feature-map cells)
    uint32_t r_cap = 0, e_cap = 0, acc_cols = 0;
    uint32_t stages = 2;     // depth of the per-warp cp.async ring of query-feature rounds
    uint32_t col_cap = 0;    // widest column range: wider chunks are cut into ranges ("virtual chunks"), each with its own image
    uint32_t n_vc = 0;       // virtual chunks of the layer
    const uint32_t* vc_ptr = nullptr;  // DEVICE [n_chunks + 1]: first virtual chunk of every chunk
    uint32_t warps_fit = 0;  // warps of the score kernel that fit next to one image in shared memory
    uint32_t off_lookup = 16, off_pre = 0, off_rp = 0, off_ew = 0, off_ec = 0;  // byte offsets inside an image
    uint32_t img_bytes = 0;  // image stride (multiple of 128)
};

// Device view of a batch of queries (either CSR or row-major dense).
struct QueryDev {
    const uint64_t* row_ptr;  // CSR: absolute offsets (row_ptr[r] - nnz_base indexes col_idx/val); nullptr for dense
    const uint32_t* col_idx;
    const float* val;         // CSR values, or the dense matrix
    uint64_t nnz_base;
    uint32_t rows;
    uint32_t cols;
    uint32_t max_row_nnz;     // longest row of the batch (sizes the shared-memory staging of the query)
};

struct XLinearStats {  // algorithmic-byte counters of SURVEY.md section 8(d), accumulated by the STATS kernel variant
    unsigned long long chunks;      // (query, chunk) products evaluated
    unsigned long long chunk_rows;  // sum R_p
    unsigned long long matched;     // sum m(q,p)   (bias row included when applied)
    unsigned long long entries;     // sum e(q,p)
    unsigned long long out_cols;    // sum c_p
    unsigned long long query_nnz;   // sum nnz(x_q) (once per query per layer)
    unsigned long long beam_out;    // sum min(k, candidates)
};

struct XLinearLayerProfile {
    double scores_ms = 0.0;  // score kernel of the layer
    double topk_ms = 0.0;    // top-k kernel of the layer
    uint64_t launches = 0;
    int scores_kernel = 0;   // last launch: 0 row-list streaming, 1 feature-map lookup, 2 dense, 3 query-warp, 4 chunk-major
    int topk_kernel = 0;     // last launch: 0 block-wide sort, 1 warp arg-max, 2 estimate filter
};

// Beam limits of a prediction, from the host model alone (no CUDA calls).  The beam entering a layer that selects a top-k
// may hold at most kXlBeamMaxTopk nodes: the block top-k keeps 2048 sort keys and three words per beam slot in <= 200 KB
// of shared memory, (200 KB - 16 KB - 4) / 12 = 15,701.  Without a top-k (selected outputs) the limit is kXlBeamMax.
// b_in, topk: as for XLinearEngine::make_plan_.
constexpr uint32_t kXlBeamMaxTopk = 15701;
constexpr uint32_t kXlBeamMax = 32768;
struct XLinearBeamCheck {
    bool fits = true;
    uint32_t layer = 0;   // first layer whose entering beam is too wide (when !fits)
    uint32_t b_prev = 0;  // that beam's width
    uint32_t limit = 0;   // the limit it exceeds
    uint32_t widest = 0;  // widest beam_size whose plan fits (0: none; 0xFFFFFFFF: every beam_size fits)
};
XLinearBeamCheck xlinear_check_beam(const XLinearHostModel& m, uint32_t beam_size, uint32_t only_topk,
                                    const std::vector<uint32_t>& b_in = {}, bool topk = true);
// Width of a result row of a (beam_size, only_topk) prediction: the last layer's k_cap in make_plan_, max(1, min(k, beam
// entering the leaf x its widest chunk)).  It is also the stride of the index-sharded exchange records.  Host model only.
uint32_t xlinear_plan_stride(const XLinearHostModel& m, uint32_t beam_size, uint32_t only_topk);

class XLinearEngine {
public:
    XLinearEngine(std::unique_ptr<XLinearHostModel> host, int device);
    ~XLinearEngine();

    const XLinearHostModel& host() const { return *host_; }
    int device() const { return device_; }

    struct Result {  // fixed-stride top-k per query, host side (pinned)
        uint32_t rows = 0;
        uint32_t stride = 0;
        uint32_t out_cols = 0;
        const uint32_t* ids = nullptr;
        const float* vals = nullptr;
        const uint32_t* cnt = nullptr;
    };

    // Host-buffer entry points (H2D + kernels + D2H inside).
    Result predict(const HostMatrix& x, uint32_t beam_size, const char* post_processor, uint32_t only_topk);

    // One layer of the python prediction chain (c_xlinear_single_layer_predict_*, pecos/core/libpecos.cpp:201-235): the
    // engine must hold a one-layer model.  codes: the previous layer's prediction as CSR rows x n_chunks, consumed in stored
    // order (no row_ptr: ones(rows x n_chunks), no combine).
    Result predict_single_layer(const HostMatrix& x, const HostMatrix& codes, const char* post_processor, uint32_t only_topk);

    // predict_on_selected_outputs (c_xlinear_predict_on_selected_outputs_*, pecos/core/libpecos.cpp:179-198): scores of exactly
    // the (query, label) pairs of the CSR pattern `sel` (rows x nr_labels), pushed through the hierarchy, no top-k.
    // Result rows have the selected rows' lengths; entry order = the reference's (see predict_selected in xlinear_engine.cu).
    // codes (one-layer models only): as for predict_single_layer.
    struct SelectedResult {
        uint32_t rows = 0, cols = 0;
        std::vector<uint64_t> indptr;
        std::vector<uint32_t> indices;
        std::vector<float> data;
    };
    SelectedResult predict_selected(const HostMatrix& x, const HostMatrix& sel, const char* post_processor,
                                    const HostMatrix& codes = {});

    // Device-resident queries (bench "value" leg: inputs already in HBM when the timed region starts).
    void resident_upload_csr(const HostMatrix& x);
    // Runs all layers over the resident batch; results stay in HBM (fetch with resident_fetch). Returns device ms.
    double resident_predict(uint32_t beam_size, const char* post_processor, uint32_t only_topk, bool collect_stats);
    Result resident_fetch();

    // Index sharding (leaf layer split over `world` GPUs, SURVEY 8e).  sharded_local_csr_packed runs every layer on this
    // GPU's shard and writes the LOCAL top-k into the caller-owned device buffer rec_dev (the NCCL all-gather send buffer)
    // as 16-byte {u64 key, u32 id, f32 value} records [rows][stride] (key == 0: empty slot), so the exchange is a single
    // all-gather; returns the stride used.  sharded_merge_packed reduces the gathered [world][rows][stride] records to the
    // global top-k.
    uint32_t sharded_local_csr_packed(const HostMatrix& x, uint32_t beam_size, const char* post_processor, uint32_t only_topk,
                                      uint32_t stride_capacity, void* rec_dev);
    Result sharded_merge_packed(uint32_t world, uint32_t rows, uint32_t stride, uint32_t only_topk, const void* g_rec);

    void set_profile(bool on) { profile_ = on; }
    // Kernel selection for A/B runs and cross-checks, described at pick_kernels_ (xlinear_engine.cu); any other value behaves as 1.
    enum class KernelMode : int { kFirstGeneration = 0, kDefault = 1, kNoQueryWarp = 2, kQueryWarpWherever = 3, kNoTopkFilter = 4,
                                  kChunkMajorWherever = 5, kQueryMajorOnly = 6, kNoPrefix = 7 };
    void set_kernel_mode(int mode) { mode_ = mode >= 0 && mode <= 7 ? static_cast<KernelMode>(mode) : KernelMode::kDefault; }
    bool has_feature_maps() const;
    // chunk-major image geometry chosen at load time for layer d (d < 0: the prefix image); ok == false: no images
    const CmShape* cm_shape_of(int d) const {
        if (d < 0) return &prefix_.cm_shape;
        return static_cast<size_t>(d) < layers_.size() ? &layers_[d].cm_shape : nullptr;
    }
    const std::vector<XLinearLayerProfile>& layer_profile() const { return layer_profile_; }
    void reset_profile();
    const std::vector<XLinearStats>& layer_stats() const { return layer_stats_; }
    uint64_t launches() const { return launches_; }
    uint64_t model_bytes() const { return model_bytes_; }

private:
    struct LayerPlan {
        uint32_t k = 0;       // only_topk used for this layer
        uint32_t b_prev = 0;  // beam capacity entering the layer
        uint32_t k_cap = 0;   // beam capacity leaving the layer
        PostProc pp;
    };
    struct LayerStore {
        DeviceBuffer<ChunkHeader> chunks;
        DeviceBuffer<uint32_t> meta;
        DeviceBuffer<uint32_t> rowext;
        DeviceBuffer<uint2> entries;
        DeviceBuffer<uint32_t> label_of_col;
        DeviceBuffer<uint2> featmap;
        DeviceBuffer<unsigned char> cm_images;  // packed chunk images of the chunk-major kernel
        DeviceBuffer<uint32_t> cm_vc_ptr;
        CmShape cm_shape;  // ok: the store has chunk images
        LayerDev view{};   // view.featmap != nullptr: the store has a feature map
    };
    // Uploads H's chunks, meta, entries and (when reordered) label_of_col into S, sets S.view from H and counts the bytes.
    void upload_store_(const ChunkedLayerHost& H, LayerStore& S);
    // Builds S's chunk images of the given shape from its view (vc_ptr: the host table of cm_layer_layout) and counts them.
    void place_images_(LayerStore& S, CmShape shape, const std::vector<uint32_t>& vc_ptr);

    // Where the last layer of a tile writes its top-k: rows [0, tile) of these arrays (keys only in an index-sharded run).
    struct OutTarget {
        uint32_t* ids;
        float* vals;
        uint32_t* cnt;
        unsigned long long* keys;
        uint32_t stride;
        OutTarget at(uint32_t row) const {
            const uint64_t o = static_cast<uint64_t>(row) * stride;
            return {ids + o, vals + o, cnt + row, keys ? keys + o : nullptr, stride};
        }
    };
    // Query rows on the device; place() is the engine's only copy of host query rows.
    struct QueryStage {
        DeviceBuffer<uint64_t> row_ptr;
        DeviceBuffer<uint32_t> col_idx;
        DeviceBuffer<float> val;  // CSR values, or the dense rows
        // placed rows are on the device (copy stream); the kernels reading them are issued (compute stream)
        cudaEvent_t landed = nullptr, consumed = nullptr;
        // room for `rows` rows of x holding n values (CSR non-zeros, or rows x cols); reallocating drops the placed rows
        void reserve(const HostMatrix& x, uint32_t rows, uint64_t n);
        // Rows [r0, r0 + tr) of x as the kernels take them, in a stage that holds x's rows from row `first` on (CSR offsets
        // stay absolute: nnz_base = x.row_ptr[first]); place() first copies them there on `stream`.
        QueryDev view(const HostMatrix& x, uint32_t first, uint32_t r0, uint32_t tr) const;
        QueryDev place(const HostMatrix& x, uint32_t first, uint32_t r0, uint32_t tr, cudaStream_t stream);
    };
    struct ResultBuffers { DeviceBuffer<uint32_t> ids, cnt; DeviceBuffer<float> vals; };  // device result rows of a call
    // for_each_tile_'s callback: layers [d_begin, d_end) over rows [r0, r0 + q.rows) of the batch, held in workspace rows
    // from ws_row on
    struct Tile { QueryDev q; uint32_t r0, ws_row; size_t d_begin, d_end; };
    using TileFn = std::function<void(const Tile& t)>;
    using BeamFn = std::function<uint32_t(uint32_t row, uint32_t* ids, float* vals)>;

    // b_in[d] (where given and > 0): the beam capacity entering layer d, set by the caller (single layer: the codes rows or
    // every parent; selected outputs: the previous layer's entry lists); otherwise the previous layer's k_cap (root: 1).
    // topk = false: no top-k kernel runs on the plan (selected outputs).
    std::vector<LayerPlan> make_plan_(uint32_t beam_size, const char* post_processor, uint32_t only_topk,
                                      const std::vector<uint32_t>& b_in = {}, bool topk = true) const;
    // Sizes the tiles of a `rows`-query call so that the workspace of one tile stays within PB200_WORKSPACE_MB, allocates
    // that workspace and returns the tile's rows.  dense_cols > 0: dense queries, whose staged tile is also capped at 4 GiB.
    uint32_t ensure_workspace_(const std::vector<LayerPlan>& plan, uint32_t rows, uint32_t dense_cols);
    // The one pass over a batch of queries x (host CSR or dense; nullptr: the resident batch) in tiles of at most `tile` rows
    // (from ensure_workspace_): stages each and hands it to run().  split: predict's CSR schedules (see the definition).
    void for_each_tile_(uint32_t tile, const HostMatrix* x, const TileFn& run, bool split = false);
    // The beam entering the first layer of a tile (rows [0, rows) of beam_*_[0]), from fill(row, ids, vals) = its length;
    // vals is nullptr unless with_vals.
    void stage_beam_(uint32_t rows, bool with_vals, const BeamFn& fill);
    // Layers [d_begin, d_end) over one tile of queries whose beam / candidate rows start at row ws_row of the workspace.
    // ext_beam: beam_*_[0] already hold the beam entering the first layer; combine_first: that layer combines its scores
    // with the beam values (single layer with a given previous prediction).
    void run_tile_(const QueryDev& q, const std::vector<LayerPlan>& plan, const OutTarget& out, uint32_t ws_row = 0,
                   bool collect_stats = false, bool ext_beam = false, int combine_first = 0, size_t d_begin = 0,
                   size_t d_end = static_cast<size_t>(-1));
    uint32_t* bid_(int b, uint32_t row) const { return beam_id_[b].get() + static_cast<uint64_t>(row) * beam_stride_; }
    float* bval_(int b, uint32_t row) const { return beam_val_[b].get() + static_cast<uint64_t>(row) * beam_stride_; }
    uint32_t* bcnt_(int b, uint32_t row) const { return beam_cnt_[b].get() + row; }
    struct TileShape;     // the facts of a call that bear on the choice of kernels (xlinear_engine.cu)
    struct LayerKernels;  // the kernels chosen for one layer of a tile (xlinear_engine.cu)
    LayerKernels pick_kernels_(size_t d, const QueryDev& q, const std::vector<LayerPlan>& plan, const TileShape& t) const;
    // The chunk-major buffers are sized, and the chunk-major score kernel may run, when the mode allows it and EVERY layer
    // has a feature map: a feature-map budget (PB200_FEATMAP_MB) that drops some layers' maps runs no layer chunk-major.
    // Letting the layers that kept their maps take it would change which kernel runs; that is for a measured change.
    bool chunk_major_workspace_() const {
        return mode_ != KernelMode::kFirstGeneration && mode_ != KernelMode::kQueryMajorOnly && has_feature_maps();
    }
    void score_layer_(size_t d, const QueryDev& q, const std::vector<LayerPlan>& plan, const LayerKernels& k, int cur,
                      uint32_t ws_row, bool collect_stats);
    OutTarget reserve_results_(ResultBuffers& r, uint32_t rows, uint32_t stride);
    Result finish_result_(const ResultBuffers& r, uint32_t rows, uint32_t stride);

    struct SelIndex {  // per layer: label -> (chunk, column offset); built on the first predict_selected call
        std::vector<uint32_t> chunk_of_label, offset_of_label;
    };
    std::vector<SelIndex> sel_index_;

    std::unique_ptr<XLinearHostModel> host_;
    int device_ = 0;
    cudaStream_t stream_ = nullptr;
    std::vector<LayerStore> layers_;
    uint64_t model_bytes_ = 0;

    // per-tile workspace
    DeviceBuffer<uint32_t> beam_id_[2];
    DeviceBuffer<float> beam_val_[2];
    DeviceBuffer<uint32_t> beam_cnt_[2];
    DeviceBuffer<float> cand_;
    DeviceBuffer<unsigned long long> sortbuf_;
    DeviceBuffer<unsigned long long> stats_dev_;
    uint32_t beam_stride_ = 0;

    // host-buffer calls: two staging sets (with copy_stream_, one is uploaded while the other is scored) and the results
    QueryStage stage_[2];
    cudaStream_t copy_stream_ = nullptr;
    ResultBuffers results_;
    PinnedBuffer<uint32_t> beam_id_host_;   // stage_beam_: the given beam, staged per tile
    PinnedBuffer<float> beam_val_host_;
    PinnedBuffer<uint32_t> beam_cnt_host_;
    // the resident batch owns its queries and results: host-buffer calls in between change neither
    QueryStage resident_stage_;
    QueryDev resident_{};
    bool has_resident_ = false;
    ResultBuffers resident_results_;
    uint32_t resident_stride_ = 0;  // top-k stride of the last resident_predict
    DeviceBuffer<unsigned long long> shard_keys_;  // local top-k of an index-sharded run before packing
    DeviceBuffer<uint32_t> shard_ids_, shard_cnt_;
    DeviceBuffer<float> shard_vals_;

    // host result staging (pinned)
    PinnedBuffer<uint32_t> out_ids_;
    PinnedBuffer<float> out_vals_;
    PinnedBuffer<uint32_t> out_cnt_;

    bool profile_ = false;
    KernelMode mode_ = KernelMode::kDefault;
    // Merged one-chunk layer of layers 0 and 1 (build_prefix_layer) and its chunk-major image: scores both layers of a tile
    // in one launch (prefix_.cm_shape.ok == false: the model is not eligible)
    LayerStore prefix_;
    // Layer 0's beam into beam_*_[1] and layer 1's raw scores into its candidate rows, for rows [ws_row, ws_row + q.rows).
    void launch_prefix_(const QueryDev& q, const std::vector<LayerPlan>& plan, uint32_t ws_row);
    uint32_t n_sm_ = 132;
    DeviceBuffer<uint32_t> cm_slot_pos_, cm_count_, cm_claim_, cm_active_, cm_bucket_ptr_, cm_pair_q_, cm_pair_pos_;
    DeviceBuffer<uint64_t> cm_cost_ptr_;
    std::vector<XLinearLayerProfile> layer_profile_;
    std::vector<XLinearStats> layer_stats_;
    uint64_t launches_ = 0;
    cudaEvent_t ev_[4] = {nullptr, nullptr, nullptr, nullptr};
};

}  // namespace pb200
