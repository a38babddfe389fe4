/*
 * pecos_b200 C ABI  --  libpecos_b200_float32.so
 *
 * Drop-in replacement, on one NVIDIA H100 (sm_90a), for the two inference hot paths that the reference exports
 * from pecos/core/libpecos.cpp and binds through ctypes in pecos/core/base.py:
 *
 *   XR-Linear beam-search prediction   (libpecos.cpp:116-176,  base.py:799-976, :990-1095)
 *   HNSW dense search                  (libpecos.cpp:449-564,  base.py:1865-1964)
 *
 * The `c_*` entry points below have byte-identical signatures, argument meaning and ownership rules to the reference
 * symbols of the same name, so `pecos.core.base.corelib` can bind them unchanged (see INTEGRATION.md).
 * The `pb200_*` entry points are additions (device selection, device-resident batches for benchmarking, profiling
 * counters, host-only model inspection for tests).
 *
 * Conventions (same as the reference): no error codes.  The reference lets C++ exceptions escape `extern "C"`
 * (=> std::terminate); this library prints the message to stderr and calls abort().  There is NO CPU fallback:
 * every compute entry point requires a CUDA device and fails loudly without one.
 * `threads` arguments are accepted and ignored (the GPU schedules the work).
 */
#ifndef PECOS_B200_H_
#define PECOS_B200_H_

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---- plain-C views of scipy/numpy buffers: pecos/core/utils/matrix.hpp:43-73, ctypes mirrors base.py:177-310 ---- */
typedef struct {
    uint32_t rows, cols;
    uint64_t* col_ptr;
    uint32_t* row_idx;
    float* val;
} ScipyCscF32;

typedef struct {
    uint32_t rows, cols;
    uint64_t* row_ptr;
    uint32_t* col_idx;
    float* val;
} ScipyCsrF32;

typedef struct {
    uint32_t rows, cols;
    float* val; /* row-major */
} ScipyDrmF32;

/* Result allocator callback (matrix.hpp:47; Python side base.py:407-478):
 *   pred_alloc(is_col_major=false, rows, cols, nnz, &indices /u32[nnz]/, &indptr /u64[rows+1]/, &data /f32[nnz]/)
 * Called exactly once per predict call, from the calling thread. */
typedef void (*py_sparse_allocator_t)(bool, uint64_t, uint64_t, uint64_t, void*, void*, void*);

/* ======================================= XR-Linear (reference-compatible) ======================================= */

/* libpecos.cpp:116  model_path = the `ranker/` folder of an XLinearModel; default layer type. */
void* c_xlinear_load_model_from_disk(const char* model_path);
/* libpecos.cpp:121  weight_matrix_type in {0 CSC, 1 HASH_CHUNKED, 2 BINARY_SEARCH_CHUNKED} (base.py:49).
 * All three are served by the one HBM chunk layout; the requested type is remembered and reported back by
 * c_xlinear_get_layer_type (pecos/xmc/base.py:1736-1743 gates features on it).  Rejects mmap folders. */
void* c_xlinear_load_model_from_disk_ext(const char* model_path, int weight_matrix_type);
/* libpecos.cpp:128  folder written by c_xlinear_compile_mmap_model (W/C/perm.mmap_store per layer). */
void* c_xlinear_load_mmap_model_from_disk(const char* model_path, const bool lazy_load);
/* libpecos.cpp:140 */
/* libpecos.cpp:133-138  npz model folder (ranker/) -> the reference's mmap format (param.json with is_mmap = true; per layer
 * W.mmap_store = chunked matrix, C.mmap_store, perm.mmap_store when the tree is not contiguously ordered; formats: SURVEY.md
 * Appendix B).  Host-only: needs no GPU.  The output loads in the reference library and here. */
void c_xlinear_compile_mmap_model(const char* model_path, const char* mmap_model_path);
void c_xlinear_destruct_model(void* ptr);
/* libpecos.cpp:147  attr in {"depth","nr_features","nr_labels","nr_codes"} (inference.hpp:2367-2379). */
uint32_t c_xlinear_get_int_attr(void* ptr, const char* attr);
/* libpecos.cpp:152 */
int c_xlinear_get_layer_type(void* ptr, int layer_depth);
/* libpecos.cpp:158-175  0 / NULL overrides mean "use the value stored with each layer". */
void c_xlinear_predict_csr_f32(void* ptr, const ScipyCsrF32* input_x, const uint32_t overridden_beam_size,
                               const char* overridden_post_processor_str, const uint32_t overridden_only_topk,
                               const int threads, py_sparse_allocator_t pred_alloc);
/* libpecos.cpp:176 */
void c_xlinear_predict_drm_f32(void* ptr, const ScipyDrmF32* input_x, const uint32_t overridden_beam_size,
                               const char* overridden_post_processor_str, const uint32_t overridden_only_topk,
                               const int threads, py_sparse_allocator_t pred_alloc);

/* libpecos.cpp:179-198  predict_on_selected_outputs: scores of exactly the (query, label) pairs of the CSR pattern
 * selected_outputs_csr (rows x nr_labels; values ignored), pushed through the hierarchy (transform + combine per layer), no
 * top-k (HierarchicalMLModel::predict_on_selected_outputs, pecos/core/xmc/inference.hpp:2507-2571).  Result: CSR with the
 * selected rows' lengths; a row's entries come in the reference's order (parents in the previous layer's order, children
 * in C's column order); labels without a path to the root leave zero entries at the row's end, like the reference.
 * The reference serves this from CSC layers only (inference.hpp:2143-2147; its Python gates on get_layer_type == CSC):
 * here every handle can, and the arithmetic is the beam-search kernels' (bit-identical raw scores). */
void c_xlinear_predict_on_selected_outputs_csr_f32(void* ptr, const ScipyCsrF32* X, const ScipyCsrF32* selected_outputs_csr,
                                                   const char* overridden_post_processor_str, const int threads,
                                                   py_sparse_allocator_t pred_alloc);
void c_xlinear_predict_on_selected_outputs_drm_f32(void* ptr, const ScipyDrmF32* X, const ScipyCsrF32* selected_outputs_csr,
                                                   const char* overridden_post_processor_str, const int threads,
                                                   py_sparse_allocator_t pred_alloc);

/* libpecos.cpp:32-36  one npz layer folder (param.json + W.npz [+ C.npz]) -> the single-layer mmap format read by
 * c_mlmodel_load_mmap_model (MLModel<csc_t>::save_mmap, inference.hpp:2274-2289).  Host-only, needs no GPU. */
void c_mlmodel_compile_mmap_model(const char* model_path, const char* mmap_model_path);
/* libpecos.cpp:37-113  Single-layer handles over ONE mmap-format MLModel folder (MLModel<csc_t>::save_mmap,
 * pecos/core/xmc/inference.hpp:2274-2289: param.json with is_mmap = true + W.mmap_store + C.mmap_store in csc_t's mmap
 * format, pecos/core/utils/matrix.hpp:386-407).  c_mlmodel_get_int_attr: nr_labels | nr_codes | nr_features.
 * c_mlmodel_predict_*: csr_codes = previous layer's prediction or NULL (= ones(rows x nr_codes), no combine);
 * overridden_post_processor NULL / overridden_only_topk 0 = the values stored with the layer.
 * Folders written by this library's or by the reference's c_mlmodel_compile_mmap_model are interchangeable. */
void* c_mlmodel_load_mmap_model(const char* model_path, const bool lazy_load);
void c_mlmodel_destruct_model(void* ptr);
uint32_t c_mlmodel_get_int_attr(void* ptr, const char* attr);
void c_mlmodel_predict_csr_f32(void* ptr, const ScipyCsrF32* input_x, const ScipyCsrF32* csr_codes,
                               const char* overridden_post_processor, const uint32_t overridden_only_topk, const int num_threads,
                               py_sparse_allocator_t pred_alloc);
void c_mlmodel_predict_drm_f32(void* ptr, const ScipyDrmF32* input_x, const ScipyCsrF32* csr_codes,
                               const char* overridden_post_processor, const uint32_t overridden_only_topk, const int num_threads,
                               py_sparse_allocator_t pred_alloc);
void c_mlmodel_predict_on_selected_outputs_csr_f32(void* ptr, const ScipyCsrF32* input_x, const ScipyCsrF32* selected_outputs_csr,
                                                   const ScipyCsrF32* csr_codes, const char* overridden_post_processor,
                                                   const int num_threads, py_sparse_allocator_t pred_alloc);
void c_mlmodel_predict_on_selected_outputs_drm_f32(void* ptr, const ScipyDrmF32* input_x, const ScipyCsrF32* selected_outputs_csr,
                                                   const ScipyCsrF32* csr_codes, const char* overridden_post_processor,
                                                   const int num_threads, py_sparse_allocator_t pred_alloc);

/* libpecos.cpp:201-235  One layer of the python prediction chain (pecos/xmc/base.py:890-949, is_predict_only=False
 * models): W ((nr_features [+1 bias row]) x nr_labels) and C (nr_labels x nr_codes) are handed over on every call;
 * csr_codes = the previous layer's prediction (rows x nr_codes, entries consumed in stored order) or NULL for the first
 * layer (= ones, no combine).  post_processor_str must be given; only_topk as passed (0 keeps nothing, like the
 * reference).  The chunked HBM layout of (W, C, bias) is built on first use and kept in a small LRU cache keyed by the
 * matrices' shapes, value pointer and a sampled content fingerprint (PB200_LAYER_CACHE entries, default 8): the
 * matrices are assumed immutable while cached (pb200_layer_cache_clear() drops them).
 * Tested in tests/test_single_layer_gpu.py; oracle pinned against the reference in tests/test_oracle_cpu.py. */
void c_xlinear_single_layer_predict_csr_f32(const ScipyCsrF32* input_x, const ScipyCsrF32* csr_codes, ScipyCscF32* W,
                                            ScipyCscF32* C, const char* post_processor_str, const uint32_t only_topk,
                                            const int num_threads, const float bias, py_sparse_allocator_t pred_alloc);
void c_xlinear_single_layer_predict_drm_f32(const ScipyDrmF32* input_x, const ScipyCsrF32* csr_codes, ScipyCscF32* W,
                                            ScipyCscF32* C, const char* post_processor_str, const uint32_t only_topk,
                                            const int num_threads, const float bias, py_sparse_allocator_t pred_alloc);
/* libpecos.cpp:238-273  the same single layer, scores of exactly the (query, label) pairs of selected_outputs_csr
 * (MLModel::predict_on_selected_outputs, inference.hpp:2129-2224; pecos/xmc/base.py:1003 = predict_on_selected_outputs of
 * is_predict_only=False models).  Result: the pattern of selected_outputs_csr, values = transformed (+ combined) scores. */
void c_xlinear_single_layer_predict_on_selected_outputs_csr_f32(const ScipyCsrF32* input_x, const ScipyCsrF32* selected_outputs_csr,
                                                                const ScipyCsrF32* csr_codes, ScipyCscF32* W, ScipyCscF32* C,
                                                                const char* post_processor_str, const int num_threads,
                                                                const float bias, py_sparse_allocator_t pred_alloc);
void c_xlinear_single_layer_predict_on_selected_outputs_drm_f32(const ScipyDrmF32* input_x, const ScipyCsrF32* selected_outputs_csr,
                                                                const ScipyCsrF32* csr_codes, ScipyCscF32* W, ScipyCscF32* C,
                                                                const char* post_processor_str, const int num_threads,
                                                                const float bias, py_sparse_allocator_t pred_alloc);
/* drops every cached single-layer engine; returns how many were held */
uint32_t pb200_layer_cache_clear(void);
/* out[0] = entries held, out[1] = hits, out[2] = misses (builds) since load */
void pb200_layer_cache_info(uint64_t* out);

/* ========================================= HNSW (reference-compatible) ========================================== */

/* libpecos.cpp:471-480  model_dir = ".../c_model" holding config.json + index.mmap_store (hnsw.hpp:534-552). */
void* c_ann_hnsw_load_drm_ip_f32(const char* model_dir, const bool lazy_load);
void* c_ann_hnsw_load_drm_l2_f32(const char* model_dir, const bool lazy_load);
/* libpecos.cpp:492-499 */
void c_ann_hnsw_destruct_drm_ip_f32(void* model_ptr);
void c_ann_hnsw_destruct_drm_l2_f32(void* model_ptr);
/* libpecos.cpp:501-524  opaque scratch pool; here: pre-allocated per-query device scratch. */
void* c_ann_hnsw_searchers_create_drm_ip_f32(void* model_ptr, uint32_t num_searcher);
void* c_ann_hnsw_searchers_create_drm_l2_f32(void* model_ptr, uint32_t num_searcher);
void c_ann_hnsw_searchers_destruct_drm_ip_f32(void* searchers_ptr);
void c_ann_hnsw_searchers_destruct_drm_l2_f32(void* searchers_ptr);
/* libpecos.cpp:527-564  caller passes zeroed Q x topk arrays; row q gets its neighbours in ascending distance. */
void c_ann_hnsw_predict_drm_ip_f32(void* model_ptr, const ScipyDrmF32* pX, uint32_t* ret_idx, float* ret_val,
                                   uint32_t efS, uint32_t topk, int32_t threads, void* searchers_ptr);
void c_ann_hnsw_predict_drm_l2_f32(void* model_ptr, const ScipyDrmF32* pX, uint32_t* ret_idx, float* ret_val,
                                   uint32_t efS, uint32_t topk, int32_t threads, void* searchers_ptr);
/* Sparse (csr) indices: HNSW<float, FeatVecSparse{IP,L2}Simd<uint32_t, float>> (libpecos.cpp:449-450, :479-480, :497-498,
 * :508-513, :522-523, :563-564; distances pecos/core/ann/feat_vectors.hpp:186-210 + distance_impl/common.hpp:15-86).  Rows of the
 * index and of the queries carry strictly ascending column indices (what scipy's sort_indices()/sum_duplicates() give and
 * the reference's block intersection assumes).  The reference's sparse "l2" evaluates to -2<x,y> (feat_vectors.hpp:186-192: the
 * squared norms are taken as do_l2_distance_simd(x, x), 0 for finite rows, NaN when a row stores a NaN or +-inf anywhere);
 * this library returns the same values, NaN for such pairs included. */
void* c_ann_hnsw_load_csr_ip_f32(const char* model_dir, const bool lazy_load);
void* c_ann_hnsw_load_csr_l2_f32(const char* model_dir, const bool lazy_load);
void c_ann_hnsw_destruct_csr_ip_f32(void* model_ptr);
void c_ann_hnsw_destruct_csr_l2_f32(void* model_ptr);
void* c_ann_hnsw_searchers_create_csr_ip_f32(void* model_ptr, uint32_t num_searcher);
void* c_ann_hnsw_searchers_create_csr_l2_f32(void* model_ptr, uint32_t num_searcher);
void c_ann_hnsw_searchers_destruct_csr_ip_f32(void* searchers_ptr);
void c_ann_hnsw_searchers_destruct_csr_l2_f32(void* searchers_ptr);
void c_ann_hnsw_predict_csr_ip_f32(void* model_ptr, const ScipyCsrF32* pX, uint32_t* ret_idx, float* ret_val,
                                   uint32_t efS, uint32_t topk, int32_t threads, void* searchers_ptr);
void c_ann_hnsw_predict_csr_l2_f32(void* model_ptr, const ScipyCsrF32* pX, uint32_t* ret_idx, float* ret_val,
                                   uint32_t efS, uint32_t topk, int32_t threads, void* searchers_ptr);

/* ============================================ pecos_b200 additions ============================================== */

const char* pb200_version(void);
/* Number of visible CUDA devices (0 when there is none; never aborts). */
int pb200_device_count(void);
/* Device used by subsequently created model handles (default 0). Returns 0 on success. */
int pb200_set_device(int device);
int pb200_get_device(void);
/* Pinned host memory for end-to-end runs (cudaMallocHost / cudaFreeHost). */
void* pb200_host_alloc(size_t bytes);
void pb200_host_free(void* ptr);
/* Overwrite a scratch buffer larger than L2 (50 MB on an H100) so the next timed iteration starts cold. */
void pb200_l2_flush(void);

/* Device-resident query batch: upload once, run the layers with inputs already in HBM, fetch when wanted.  The batch and
 * its results have their own device buffers: host-buffer calls on the same handle in between change neither. */
void pb200_xlinear_resident_upload_csr(void* ptr, const ScipyCsrF32* input_x);
/* Returns the device time (ms, CUDA events on the engine's stream) of one pass over the resident batch. */
double pb200_xlinear_resident_predict(void* ptr, uint32_t overridden_beam_size, const char* overridden_post_processor_str,
                                      uint32_t overridden_only_topk, int collect_stats);
void pb200_xlinear_resident_fetch(void* ptr, py_sparse_allocator_t pred_alloc);

/* Index sharding of the leaf layer over `shard_world` GPUs (one process per GPU; SURVEY.md 8e).  Upper layers are
 * replicated, so every rank walks the identical global beam; rank r keeps the weights of a contiguous range of leaf
 * chunks and scores only those.  weight_matrix_type < 0 loads an mmap folder.
 *   local:  runs all layers, writes this rank's top-k as 16-byte records {u64 key, u32 id, f32 value}[rows][stride] into
 *           the CALLER-OWNED DEVICE buffer rec_dev (the send buffer of ONE ncclAllGather, 16 B x rows x stride per rank);
 *           key == 0 marks an empty slot, so no count array travels.  Returns stride (<= capacity).
 *   merge:  gathered [world][rows][stride] records g_rec -> global top-k, returned through pred_alloc like
 *           c_xlinear_predict_*.
 * The result is bit-identical to the unsharded prediction (keys carry the candidate's global position). */
void* pb200_xlinear_load_sharded(const char* model_path, int weight_matrix_type, uint32_t shard_rank, uint32_t shard_world);
void pb200_xlinear_get_shard(void* ptr, uint32_t* out /* rank, world, leaf_chunk_begin, leaf_chunk_end */);
uint32_t pb200_xlinear_sharded_local_csr_packed(void* ptr, const ScipyCsrF32* input_x, uint32_t overridden_beam_size,
                                                const char* overridden_post_processor_str, uint32_t overridden_only_topk,
                                                uint32_t stride_capacity, void* rec_dev);
void pb200_xlinear_sharded_merge_packed(void* ptr, uint32_t world, uint32_t rows, uint32_t stride, uint32_t overridden_only_topk,
                                        const void* g_rec, py_sparse_allocator_t pred_alloc);

/* Per-layer kernel timing (CUDA events) and algorithmic-byte counters.
 *   profile: out[2*d] = chunk-score kernel ms, out[2*d+1] = top-k kernel ms   (accumulated since reset)
 *   stats:   out[7*d + {0..6}] = chunks, sum R, sum m, sum e, sum c, sum nnz(x), sum beam-out   (last stats pass) */
void pb200_xlinear_set_profile(void* ptr, int on);
/* Kernel mode for A/B tests (results are identical in every mode): 0 first generation (row-list streaming + block-wide
 * sort), 1 default, 2 no query-warp kernel, 3 query-warp kernel wherever it fits, 4 no top-k estimate filter, 5 chunk-major
 * kernel wherever a layer has chunk images and the prefix launch on tiles of any size, 6 query-major kernels only, 7 no
 * prefix launch.  Any other value behaves as 1.  XLinearEngine::pick_kernels_ (pecos_b200/csrc/xlinear_engine.cu) states
 * what each mode lets a layer take and the order in which the kernels are preferred.
 * Prefix launch (modes 1 - 5): a sparse tile of enough queries scores layers 0 and 1 in ONE chunk-major launch (kernel id 4
 * for both layers; layer 0's top-k slot and layer 1's score slot then read 0 ms).
 * Returns 1 when every layer has a feature map (PB200_FEATMAP_MB caps their total size at load time, default 32768). */
int pb200_xlinear_set_lookup(void* ptr, int on);
void pb200_xlinear_reset_profile(void* ptr);
void pb200_xlinear_get_profile(void* ptr, double* out);
/* out[2*depth]: per layer {score kernel, top-k kernel} of the last call.  Score: 0 row-list streaming, 1 feature-map
 * lookup (xl_chunk_scores_kernel), 2 dense, 3 xl_query_warp_scores_kernel, 4 xl_cm_scores_kernel.  Top-k: 0 xl_topk_kernel,
 * 1 xl_topk_warp_kernel, 2 xl_topk_filter_kernel. */
void pb200_xlinear_get_kernel_ids(void* ptr, int* out);
/* The chunk-major image geometry chosen at load time for `layer` (-1: the merged prefix image of layers 0 and 1):
 * out[6] = {images built, direct feature table, column cap (wider chunks are cut into ranges of at most this many columns),
 * virtual chunks, bytes per image, warps that fit next to one image}.  Returns 1 (out untouched) for a layer out of range. */
int pb200_xlinear_cm_info(void* ptr, int layer, uint64_t* out);
void pb200_xlinear_get_stats(void* ptr, uint64_t* out);
uint64_t pb200_xlinear_launches(void* ptr);
uint64_t pb200_xlinear_model_bytes(void* ptr);
/* Replicas held by a handle: 1, or one per entry of PB200_DEVICES ("0,1,..." | "all", read at load time).  With replicas a
 * c_xlinear_predict_* / c_ann_hnsw_predict_* call splits its rows over the devices (one host thread + stream each) and
 * concatenates the results in row order -- the multi-GPU form of the reference's OpenMP loop over queries
 * (pecos/core/xmc/inference.hpp:969-1005, pecos/core/libpecos.cpp:540-548). */
uint32_t pb200_xlinear_replicas(void* ptr);
uint32_t pb200_hnsw_replicas(void* model_ptr);

/* HNSW: device-resident query batch (its queries and results survive host-buffer calls on the same handle), search-kernel
 * time (ms, CUDA events), algorithmic counters of the last search
 *   counters out[4] = {distance evaluations, level-0 expansions, upper-level neighbourhood reads, queries}
 *   info     out[8] = {num_node, feat_dim, maxM, maxM0, max_level, init_node, index bytes in HBM, kernel launches} */
void pb200_hnsw_resident_upload(void* model_ptr, const ScipyDrmF32* pX);
double pb200_hnsw_resident_predict(void* model_ptr, uint32_t efS, uint32_t topk);
void pb200_hnsw_resident_fetch(void* model_ptr, uint32_t* ret_idx, float* ret_val);
void pb200_hnsw_get_counters(void* model_ptr, uint64_t* out);
/* sparse (csr) indices: resident csr batch; stored entries (8 bytes each) of the base rows evaluated by the last search */
void pb200_hnsw_resident_upload_csr(void* model_ptr, const ScipyCsrF32* pX);
uint64_t pb200_hnsw_sparse_entries(void* model_ptr);
/* HNSW index sharding (pecos_b200.hnsw_build.build_hnsw_shards: one independent index per contiguous row range, one process
 * per GPU).  model_ptr is a c_ann_hnsw_load_* handle of this rank's shard; only its primary engine is used.
 *   local:  searches the shard and writes its top-k as 16-byte records {u64 key, u32 id, f32 value}[rows][topk] into the
 *           CALLER-OWNED DEVICE buffer rec_dev (the send buffer of ONE all-gather).  id = id_offset + local id (the shard's
 *           first global row), value = distance, key = (~orderable(distance) << 32) | ~(rank * topk + slot), where every NaN
 *           takes orderable = 0xFFFFFFFF whatever its sign and payload; key 0 marks an empty slot.  Requires
 *           (rank + 1) * topk <= 1024.
 *   merge:  gathered [world][rows][topk] records g_rec -> ret_idx / ret_val [rows][topk] (host), ordered by (distance with
 *           NaN last, shard rank, slot); rows with fewer than topk results end in zeros, like c_ann_hnsw_predict_*.
 *           Requires world * topk <= 1024.
 * The result equals, bit for bit, the merge by that order of the per-shard c_ann_hnsw_predict_* results.  At world 1 this
 * is the unsharded search when no NaN is returned; otherwise it is the unsharded search's entries ordered by (distance with
 * NaN last, position): a NaN in the search heaps can leave the unsharded result out of order, and the merge sorts it. */
void pb200_hnsw_sharded_local_packed_drm(void* model_ptr, const ScipyDrmF32* pX, uint32_t efS, uint32_t topk, uint32_t rank,
                                         uint32_t id_offset, void* rec_dev);
void pb200_hnsw_sharded_local_packed_csr(void* model_ptr, const ScipyCsrF32* pX, uint32_t efS, uint32_t topk, uint32_t rank,
                                         uint32_t id_offset, void* rec_dev);
void pb200_hnsw_sharded_merge_packed(void* model_ptr, uint32_t world, uint32_t rows, uint32_t topk, const void* g_rec,
                                     uint32_t* ret_idx, float* ret_val);
/* libpecos.cpp:482-490  c_ann_hnsw_save_drm_{ip,l2}_f32(model_ptr, model_dir): for an index loaded by THIS library the saved
 * form is what it was loaded from (config.json + index.mmap_store are copied to model_dir).
 *
 * Handles are library-specific: an index TRAINED by the reference (c_ann_hnsw_train_* is not served here) is a reference
 * handle, but after the overlay the reference's Python passes it to this library's destruct / searchers / predict / save.
 * pb200_hnsw_set_foreign registers the reference's own functions for one index type (0 = drm ip, 1 = drm l2, 2 = csr ip, 3 = csr l2); handles and searcher tokens
 * that were not created here are forwarded to them (pecos_b200.integration.overlay does this).  Without the registration a
 * foreign handle is a fatal error with a clear message. */
void c_ann_hnsw_save_drm_ip_f32(void* model_ptr, const char* model_dir);
void c_ann_hnsw_save_drm_l2_f32(void* model_ptr, const char* model_dir);
void c_ann_hnsw_save_csr_ip_f32(void* model_ptr, const char* model_dir);
void c_ann_hnsw_save_csr_l2_f32(void* model_ptr, const char* model_dir);
void pb200_hnsw_set_foreign(int metric, void* destruct, void* searchers_create, void* searchers_destruct, void* predict, void* save);

/* ================================================== PairwiseANN ================================================== */
/* libpecos.cpp:567-659, pecos/core/ann/pairwise.hpp.  Two types, as in the reference: drm (dense X_trn, FeatVecDenseIPSimd) and
 * csr (X_trn rows with strictly ascending indices, FeatVecSparseIPSimd); inner-product distance only.
 * train deep-copies X_trn and Y_csc (X.rows must equal Y.rows); load reads <model>/c_model (config.json + index.mmap_store) and
 * save writes the same two files.  Neither touches the GPU: a model's arrays move to the device on its first search.
 * searchers_create: num_searcher is accepted and ignored; a token owns a stream and scratch, calls on one token are
 * serialised, tokens of one model may run concurrently.
 * predict: pair b uses query row (is_same_input ? 0 : b) and column label_keys[b]; slot k < min(only_topk, column length)
 * of row b of ret_* (batch_size x only_topk) receives {row id, distance, Y value, 1} in the reference's order, ties
 * included; every other slot is left as the caller had it.  A label key >= the model's number of labels, or a dense model
 * wider than pb200_pairwise_ann_dense_fits allows, is a fatal error before any GPU work.  NaN distances (a NaN component, or
 * products that overflow to both +inf and -inf) are placed where the reference's heap sequence puts them. */
void* c_pairwise_ann_train_drm_ip_f32(const ScipyDrmF32* pX, const ScipyCscF32* pY);
void* c_pairwise_ann_train_csr_ip_f32(const ScipyCsrF32* pX, const ScipyCscF32* pY);
void* c_pairwise_ann_load_drm_ip_f32(const char* model_dir, const bool lazy_load);
void* c_pairwise_ann_load_csr_ip_f32(const char* model_dir, const bool lazy_load);
void c_pairwise_ann_save_drm_ip_f32(void* model_ptr, const char* model_dir);
void c_pairwise_ann_save_csr_ip_f32(void* model_ptr, const char* model_dir);
void c_pairwise_ann_destruct_drm_ip_f32(void* model_ptr);
void c_pairwise_ann_destruct_csr_ip_f32(void* model_ptr);
void* c_pairwise_ann_searchers_create_drm_ip_f32(void* model_ptr, uint32_t num_searcher);
void* c_pairwise_ann_searchers_create_csr_ip_f32(void* model_ptr, uint32_t num_searcher);
void c_pairwise_ann_searchers_destruct_drm_ip_f32(void* searchers_ptr);
void c_pairwise_ann_searchers_destruct_csr_ip_f32(void* searchers_ptr);
void c_pairwise_ann_predict_drm_ip_f32(void* searchers_ptr, uint32_t batch_size, uint32_t only_topk, const ScipyDrmF32* pQ,
                                       uint32_t* label_keys, uint32_t* ret_Imat, uint32_t* ret_Mmat, float* ret_Dmat,
                                       float* ret_Vmat, const bool is_same_input);
void c_pairwise_ann_predict_csr_ip_f32(void* searchers_ptr, uint32_t batch_size, uint32_t only_topk, const ScipyCsrF32* pQ,
                                       uint32_t* label_keys, uint32_t* ret_Imat, uint32_t* ret_Mmat, float* ret_Dmat,
                                       float* ret_Vmat, const bool is_same_input);
/* the token's last predict call: out[4] = {pairs, distances evaluated (sum of column lengths), stored entries of the sparse
 * rows read, pairs whose selection replayed the reference's heap sequence (ties at the top-k boundary or within it)} */
void pb200_pairwise_ann_get_counters(void* searchers_ptr, uint64_t* out);
/* device time (CUDA events) of the distance and select kernels of the token's last predict call, in ms */
double pb200_pairwise_ann_kernel_ms(void* searchers_ptr);
/* the token's last predict call: out[4] = {bulk-copy ring depth of the distance kernel (4, or 0 = direct loads), warps per
 * CTA, shared-memory bytes per warp, tiles (consecutive pairs whose columns hold at most 2^25 entries together, or one longer
 * column)}; all 0 when the call had nothing to search (batch_size or only_topk 0) */
void pb200_pairwise_ann_launch_info(void* searchers_ptr, uint64_t* out);
/* Width limit of dense models, host-only.  A warp of the distance kernel stages the query row (dense_vstride(d) floats: d
 * rounded up to 64 when d % 16 == 0, else the 16-multiple part rounded up to 64 plus 16) and the distances of 128 rows in
 * 200 KB of shared memory, with a ring of 4 more rows where that fits (d <= 10,191).  Every d up to 51,024 and every multiple
 * of 16 up to 51,072 fits; nothing else does, and predict on such a model is a fatal error, so callers check first (the Python
 * layer raises ValueError).  Training, saving and loading a wider model are allowed.  Returns 1 if a model of width feat_dim
 * can be searched, else 0, and out[3] = {ring depth (4 or 0), per-warp bytes at that depth, row stride in floats}. */
int pb200_pairwise_ann_dense_fits(uint32_t feat_dim, uint32_t* out);
/* Host-only ingest check of a PairwiseANN folder (<model>/c_model), no GPU needed: pairwise_ann_t of the data type (sparse 0 =
 * drm, 1 = csr), version, block sizes, offsets, row ids of Y within X.  Returns 0 and out[6] = {num_input_keys, num_label_keys,
 * feat_dim, nnz of Y, nnz of X, longest column}, or 1 (reason on stderr). */
int pb200_pairwise_ann_host_info(const char* model_dir, int sparse, uint64_t* out);

/* ============================================ sparse x sparse products ============================================ */
/* libpecos.cpp:320-335, smat_x_smat (pecos/core/utils/matrix.hpp:1062-1290).  csr: Z = X Y, row i of Z from row i of X and
 * the rows of Y, pred_alloc(false, X.rows, Y.cols, nnz); csc: column i of Z from column i of Y and the columns of X,
 * pred_alloc(true, X.rows, Y.cols, nnz).  Bit-identical to the reference: each output entry starts at +0.0f and receives
 * acc = acc + a_s * b_t (separate roundings) for every contribution in traversal order (entries s of the A row in stored
 * order, then entries t of B row A.idx[s] in stored order); repeated and unsorted indices are separate contributions.  Indices
 * of an output row come ascending (sorted_indices) or in first-touch order.  pred_alloc gets the number of distinct indices
 * touched; with eliminate_zeros, entries equal to +-0 are then compacted out (NaN stays) and indptr describes what is left.
 * pred_alloc is called exactly once, from the calling thread, also for empty products; threads is accepted and ignored.
 * X.cols != Y.rows, an index of the left operand (csr: X, csc: Y) beyond the right operand's rows, or one of the right operand
 * beyond the output width is a fatal error before any GPU work.  Runs on the pb200_set_device device; calls on one device are
 * serialised.  The device workspace (hash accumulators, output staging, A tiles) is bounded by PB200_SPMM_WORKSPACE_MB
 * (read on every call, default 1024); a single row that needs more runs as a tile of its own. */
void c_sparse_matmul_csr_f32(const ScipyCsrF32* pX, const ScipyCsrF32* pY, py_sparse_allocator_t pred_alloc,
                             const bool eliminate_zeros, const bool sorted_indices, int threads);
void c_sparse_matmul_csc_f32(const ScipyCscF32* pX, const ScipyCscF32* pY, py_sparse_allocator_t pred_alloc,
                             const bool eliminate_zeros, const bool sorted_indices, int threads);
/* 1 if a product whose right operand (csr: Y, csc: X, as rows of the traversal) has b_rows rows and b_nnz entries fits the
 * current device: its arrays, one flag byte per row and 64 MB of workspace within cudaMemGetInfo's free bytes; else 0 (also
 * without a device).  out[2] = {bytes needed, free bytes}. */
int pb200_spmm_fits(uint32_t b_rows, uint64_t b_nnz, uint64_t* out);
/* The calling thread's last product: out[10] = {A rows (csr: X.rows, csc: Y.cols), products (sum over A entries of their B
 * row lengths), nnz handed to pred_alloc, nnz kept after eliminate_zeros, rows counted by the warp / CTA symbolic kernels,
 * rows folded by the warp / CTA numeric kernels, tiles, kernel launches}. */
void pb200_spmm_last_info(uint64_t* out);
/* device time (CUDA events) of the calling thread's last product's kernels, in ms */
double pb200_spmm_last_kernel_ms(void);

/* base-vector rows kept in flight per warp by the bulk-copy (TMA) ring: 0 = direct loads, 4 (default) or 8; returns the
 * value in effect.  Results are identical for every setting.  A search whose per-warp shared-memory slice (query + ring
 * rows + neighbour slots + result heap) would exceed 200 KB at this depth runs the next shallower one that fits
 * (8 -> 4 -> 0), and where depth 0 does not fit either, the result heap moves to global memory (as for every ef > 512). */
int pb200_hnsw_set_stages(void* model_ptr, int stages);
/* Width limit of dense indices, host-only.  With ef = max(efS, topk) and nbmax = the longest neighbour list (level 0 or
 * above) rounded up to 32, a warp's slice holds the query row (dense_vstride(d) floats, see
 * pb200_pairwise_ann_dense_fits), 8 * nbmax bytes of neighbour ids and distances, the ring rows and, while ef <= 512 and it
 * fits, the (ef + 1)-entry result heap.  A dense index is searchable for every ef iff 4 * dense_vstride(d) + 8 * nbmax
 * <= 204,800 (M = 16: every d up to 51,087 and every multiple of 16 up to 51,136); a wider one loads, saves and creates
 * searchers, but predict on it is a fatal error, so callers check first (HNSW.predict and ShardedHNSW.predict raise
 * ValueError).  Sparse indices have no width limit.  Both return 1 if the search fits, else 0, and out[5] = {ring depth,
 * result heap in shared memory (1) or global memory (0), per-warp bytes, nbmax, row stride in floats (sparse: 0)}.
 *   search_fits: for a handle at its pb200_hnsw_set_stages setting; handles of the reference library report 1, out zeros.
 *   dense_plan:  for a dense index of width feat_dim whose longest neighbour list has max_degree entries. */
int pb200_hnsw_search_fits(void* model_ptr, uint32_t efS, uint32_t topk, uint32_t* out);
int pb200_hnsw_dense_plan(uint32_t feat_dim, uint32_t max_degree, int stages, uint32_t efS, uint32_t topk, uint32_t* out);
/* the last search launch of the handle's primary engine: out[5] = {ring depth it ran, warps per CTA, CTAs, dynamic shared
 * memory per CTA in bytes, result-heap entries allocated in global scratch (heaps of ef > 512, and of the widest dense rows,
 * live there; grows only)} */
void pb200_hnsw_launch_info(void* model_ptr, uint64_t* out);
void pb200_hnsw_get_info(void* model_ptr, uint64_t* out);
/* Host-only ingest check of an HNSW index folder (<model>/c_model), no GPU needed: the loader's validation of config.json
 * (hnsw_t string of the requested metric / data type, version) and of index.mmap_store (record sizes; sparse: record offsets,
 * strictly ascending in-range indices).  metric 0 = ip, 1 = l2; sparse 0 = drm, 1 = csr.  Returns 0 and
 * out[8] = {num_node, feat_dim, maxM, maxM0, max_level, init_node, stored vector entries, level-0 degree sum}, or 1 (reason on stderr). */
int pb200_hnsw_host_info(const char* model_dir, int metric, int sparse, uint64_t* out);
/* A query whose candidate queue outgrows the per-warp scratch (PB200_HNSW_VCAP entries, default 32768) makes the engine re-run
 * the batch with twice the capacity (up to num_node + 1, which cannot overflow) -- this counts those re-runs. */
uint32_t pb200_hnsw_vcap_retries(void* model_ptr);

/* ============================================= index construction =============================================== */

/* Distance kernels of the sparse (csr) HNSW builder (pecos_b200/hnsw_build.py).  Every argument is a DEVICE pointer on
 * `device` (torch tensors' data_ptr()), work is enqueued on `stream` (a cudaStream_t, NULL = the legacy default stream) and
 * the call returns without synchronising; the caller's current device is left as it was.  metric 0 = ip, 1 = l2.
 * Base rows: row r = entries [row_ptr[r], row_ptr[r+1]) (u64) of ent, 8 bytes each {u32 index, f32 value}, indices strictly
 * ascending.  Each returned distance is bit-identical to the reference's FeatVecSparse{IP,L2}Simd::distance of the two rows
 * (ip: 1 - <x,y>; l2: -2<x,y>, see above).  work (may be NULL): a device u64 that is increased by the postings walked
 * (block) or the row entries walked by the intersections (candidate sets). */

/* Prefix-kNN blocks.  The candidate set is given by its inverted index: column f = postings [col_ptr[f], col_ptr[f+1]) (u64)
 * of post, 8 bytes each {u32 position in the candidate set, f32 value}, positions ascending within a column.
 * out (f32 [nq, nc]): out[q * nc + (p - c0)] = distance(row q_ids[q] (i64), candidate at position p), p in [c0, c0 + nc). */
void pb200_sparse_block_distances(int device, int metric, const void* row_ptr, const void* ent, const void* q_ids, uint32_t nq,
                                  const void* col_ptr, const void* post, uint32_t c0, uint32_t nc, void* out, void* work,
                                  void* stream);
/* Selection-heuristic candidate sets.  cand (i64 [n, C], C <= 512): row ids, -1 = empty slot.
 * out (f32 [n, C, C]): out[t, i, j] = distance(cand[t, i], cand[t, j]); +inf where either slot is empty. */
void pb200_sparse_candidate_distances(int device, int metric, const void* row_ptr, const void* ent, const void* cand, uint32_t n,
                                      uint32_t C, void* out, void* work, void* stream);

/* Host-only model ingest (no GPU needed): loads + builds the chunk layout, for layout tests.
 *   kind: 0 = npz folder, 1 = mmap folder.  dims out[8] = {w_rows, n_cols, out_cols, n_chunks, c_max, meta_len,
 *   n_entries, label_of_col_len}.  export copies the arrays into caller buffers (any may be NULL). */
void* pb200_xlinear_host_load(const char* model_path, int kind);
/* host-only: the one-layer model c_xlinear_single_layer_predict_* builds from in-memory W / C (same handle type) */
void* pb200_xlinear_host_from_csc(const ScipyCscF32* W, const ScipyCscF32* C, float bias);
/* host-only: a new one-layer handle holding the merged layer that scores layers 0 and 1 of hptr in one pass (W = [W0 | W1],
 * one chunk, one shared bias row); hptr must have depth >= 2, neither layer rearranged, both over the same features */
void* pb200_xlinear_host_prefix_layer(void* hptr);
void pb200_xlinear_host_free(void* hptr);
uint32_t pb200_xlinear_host_depth(void* hptr);
void pb200_xlinear_host_layer_dims(void* hptr, uint32_t layer, uint64_t* out);
void pb200_xlinear_host_layer_export(void* hptr, uint32_t layer, void* chunks32, uint32_t* meta, void* entries8,
                                     uint32_t* label_of_col);
/* Beam limit of XR-Linear prediction.  The beam entering a layer (1 at the root, then min(k, candidates) of the layer above,
 * k = beam_size or the stored only_topk) may hold at most 15,701 nodes: the block top-k keeps 2048 sort keys and three words
 * per beam slot in 200 KB of shared memory.  c_xlinear_predict_* (and the resident / index-sharded calls) with a wider beam
 * is a fatal error, so callers check first: returns 1 when the (beam_size, only_topk) call fits, else 0, and
 * out[4] = {first layer whose entering beam is too wide, that beam's width, the limit, widest beam_size that fits
 * (0xFFFFFFFF: all)}.  Host-only: hptr is a pb200_xlinear_host_* handle, ptr a loaded model (c_xlinear_load_*). */
int pb200_xlinear_host_plan_fits(void* hptr, uint32_t beam_size, uint32_t only_topk, uint32_t* out);
int pb200_xlinear_plan_fits(void* ptr, uint32_t beam_size, uint32_t only_topk, uint32_t* out);
/* Width of a result row of a (beam_size, only_topk) call: the last layer's top-k capacity max(1, min(k, beam entering the
 * leaf x its widest chunk)), k = only_topk or the stored one.  It is the stride of the index-sharded exchange records, so
 * callers check world x stride against the merge capacity (1024 records per query) before any GPU work.  Host-only: ptr is
 * a loaded model, or with host != 0 a pb200_xlinear_host_* handle. */
uint32_t pb200_xlinear_plan_stride(void* ptr, int host, uint32_t beam_size, uint32_t only_topk);
/* The limit itself: 15,701 when the layer selects a top-k (topk != 0), else 32,768.  One layer of the python chain
 * (c_xlinear_single_layer_predict_*) enters with a beam of max(row nnz of csr_codes) nodes, or C.cols without codes. */
uint32_t pb200_xlinear_beam_limit(int topk);

#ifdef __cplusplus
}
#endif
#endif /* PECOS_B200_H_ */
