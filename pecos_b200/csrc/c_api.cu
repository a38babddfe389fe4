// extern "C" boundary of libpecos_b200_float32.so: XR-Linear entry points + pb200_* additions.
// Signatures mirror pecos/core/libpecos.cpp:116-176 (see include/pecos_b200.h for the per-symbol citations).
#include "../../include/pecos_b200.h"

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <exception>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_set>
#include <vector>

#include "hnsw_build_sparse.h"
#include "hnsw_engine.h"
#include "pairwise_engine.h"
#include "spmm_engine.h"
#include "xlinear_engine.h"

namespace {

std::atomic<int> g_device{0};

[[noreturn]] void die(const char* where, const char* what) {
    std::fprintf(stderr, "pecos_b200 fatal error in %s: %s\n", where, what);
    std::fflush(stderr);
    std::abort();
}

#define PB200_API_BEGIN try {
#define PB200_API_END(name)                                  \
    }                                                        \
    catch (const std::exception& e) { die(name, e.what()); } \
    catch (...) { die(name, "unknown exception"); }

// In-library multi-GPU query fan-out (SURVEY 8e; the reference's analogue is the OpenMP loop over work items,
// pecos/core/xmc/inference.hpp:969-1005): PB200_DEVICES="0,1,2,3" | "all" at LOAD time puts a replica of the model on every
// listed device; a predict call then splits its rows into contiguous blocks balanced by nnz, one host thread + stream per
// device, and the per-device results are concatenated in row order into the single pred_alloc buffers.  A device may be
// listed more than once (two engines on one GPU: how the single-GPU tests emulate a world of 2).  Unset: one engine on the
// device chosen by pb200_set_device.
std::vector<int> device_list() {
    std::vector<int> out;
    const char* env = std::getenv("PB200_DEVICES");
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0)
        throw std::runtime_error("no CUDA device visible: pecos_b200 has no CPU fallback");
    if (!env || !*env) { out.push_back(g_device.load()); return out; }
    const std::string v(env);
    if (v == "all") { for (int i = 0; i < n; ++i) out.push_back(i); return out; }
    size_t pos = 0;
    while (pos <= v.size()) {
        const size_t comma = v.find(',', pos);
        const std::string tok = v.substr(pos, comma == std::string::npos ? std::string::npos : comma - pos);
        if (!tok.empty()) {
            char* end = nullptr;
            const long d = std::strtol(tok.c_str(), &end, 10);
            if (*end != 0 || d < 0 || d >= n) throw std::runtime_error("PB200_DEVICES: bad device id '" + tok + "'");
            out.push_back(static_cast<int>(d));
        }
        if (comma == std::string::npos) break;
        pos = comma + 1;
    }
    if (out.empty()) out.push_back(g_device.load());
    return out;
}

// runs fn(i) for i in [0, n) on n host threads (fn(0) on the caller); rethrows the first exception
template <typename F>
void fan_out(size_t n, F&& fn) {
    if (n <= 1) { if (n == 1) fn(0); return; }
    std::vector<std::exception_ptr> err(n);
    std::vector<std::thread> th;
    th.reserve(n - 1);
    for (size_t i = 1; i < n; ++i)
        th.emplace_back([&, i] { try { fn(i); } catch (...) { err[i] = std::current_exception(); } });
    try { fn(0); } catch (...) { err[0] = std::current_exception(); }
    for (auto& t : th) t.join();
    for (auto& e : err) if (e) std::rethrow_exception(e);
}

// An XR-Linear or HNSW handle.  The reference's handles are immutable after load and may be shared between threads (ctypes
// drops the GIL during a call).  Ours own device workspaces, so calls on ONE handle are serialised; different handles run
// concurrently.
template <typename Engine>
struct Replicas {
    std::vector<std::unique_ptr<Engine>> engines;  // [0] = primary; > 1: PB200_DEVICES replicas for the query fan-out
    std::mutex mu;
    Engine& primary() { return *engines.at(0); }
};

using XLinearHandle = Replicas<pb200::XLinearEngine>;

struct HnswHandle : Replicas<pb200::HnswEngine> {
    std::string model_dir;  // <model>/c_model the index was loaded from (c_ann_hnsw_save copies it)
};

XLinearHandle& xlinear_of(void* ptr) {
    if (!ptr) throw std::runtime_error("null model handle");
    return *static_cast<XLinearHandle*>(ptr);
}

HnswHandle& hnsw_of(void* ptr) {
    if (!ptr) throw std::runtime_error("null HNSW handle");
    return *static_cast<HnswHandle*>(ptr);
}

#define PB200_LOCK(handle) std::lock_guard<std::mutex> pb200_handle_lock((handle).mu);

// One engine per device of devs, built concurrently.  host_for(i) makes the host model engine i consumes while uploading; it
// runs on the calling thread from the last engine to the first, so host_for(0) may hand over the model the others copied.
template <typename Engine, typename HostFor>
void load_replicas(Replicas<Engine>& h, const std::vector<int>& devs, HostFor&& host_for) {
    std::vector<decltype(host_for(size_t{0}))> hosts(devs.size());
    for (size_t i = devs.size(); i-- > 0;) hosts[i] = host_for(i);
    h.engines.resize(devs.size());
    fan_out(devs.size(), [&](size_t i) { h.engines[i] = std::make_unique<Engine>(std::move(hosts[i]), devs[i]); });
}

// pb200_xlinear_{host_,}plan_fits: 1 if a predict call with (beam_size, only_topk) fits the beam limits, else 0;
// out[4] = {first layer whose entering beam is too wide, that beam's width, the limit, widest beam_size that fits}
int plan_fits(const pb200::XLinearHostModel& m, uint32_t beam_size, uint32_t only_topk, uint32_t* out) {
    const pb200::XLinearBeamCheck r = pb200::xlinear_check_beam(m, beam_size, only_topk);
    if (out) { out[0] = r.layer; out[1] = r.b_prev; out[2] = r.limit; out[3] = r.widest; }
    return r.fits ? 1 : 0;
}

void emit_results(const std::vector<pb200::XLinearEngine::Result>& parts, py_sparse_allocator_t pred_alloc) {
    // create_pycsr contract (pecos/core/utils/matrix.hpp:300-316): one allocator call, then fill the three arrays.
    uint64_t nnz = 0, rows = 0;
    bool all_full = true;
    for (const auto& r : parts) {
        uint64_t part = 0;
        for (uint32_t i = 0; i < r.rows; ++i) part += r.cnt[i];
        all_full = all_full && (part == static_cast<uint64_t>(r.rows) * r.stride);
        nnz += part;
        rows += r.rows;
    }
    uint32_t* indices = nullptr;
    uint64_t* indptr = nullptr;
    float* data = nullptr;
    pred_alloc(false, rows, parts.empty() ? 0 : parts[0].out_cols, nnz, &indices, &indptr, &data);
    if (!indptr || (nnz && (!indices || !data))) throw std::runtime_error("result allocator returned null buffers");
    uint64_t w = 0, row = 0;
    indptr[0] = 0;
    for (const auto& r : parts) {
        if (all_full) {
            // every row is full: the fixed-stride device layout already is the CSR payload
            const uint64_t n = static_cast<uint64_t>(r.rows) * r.stride;
            if (n) {
                std::memcpy(indices + w, r.ids, n * sizeof(uint32_t));
                std::memcpy(data + w, r.vals, n * sizeof(float));
            }
            for (uint32_t i = 0; i < r.rows; ++i) indptr[row + i + 1] = w + static_cast<uint64_t>(i + 1) * r.stride;
            w += n;
        } else {
            for (uint32_t i = 0; i < r.rows; ++i) {
                const uint32_t c = r.cnt[i];
                std::memcpy(indices + w, r.ids + static_cast<uint64_t>(i) * r.stride, c * sizeof(uint32_t));
                std::memcpy(data + w, r.vals + static_cast<uint64_t>(i) * r.stride, c * sizeof(float));
                w += c;
                indptr[row + i + 1] = w;
            }
        }
        row += r.rows;
    }
}

void emit_result(const pb200::XLinearEngine::Result& r, py_sparse_allocator_t pred_alloc) {
    emit_results(std::vector<pb200::XLinearEngine::Result>{r}, pred_alloc);
}

void emit_selected(const pb200::XLinearEngine::SelectedResult& r, py_sparse_allocator_t pred_alloc) {
    uint32_t* indices = nullptr;
    uint64_t* indptr = nullptr;
    float* data = nullptr;
    const uint64_t nnz = r.indptr.empty() ? 0 : r.indptr.back();
    pred_alloc(false, r.rows, r.cols, nnz, &indices, &indptr, &data);
    if (!indptr || (nnz && (!indices || !data))) throw std::runtime_error("result allocator returned null buffers");
    std::memcpy(indptr, r.indptr.data(), r.indptr.size() * sizeof(uint64_t));
    if (nnz) {
        std::memcpy(indices, r.indices.data(), nnz * sizeof(uint32_t));
        std::memcpy(data, r.data.data(), nnz * sizeof(float));
    }
}

void* make_engine(std::unique_ptr<pb200::XLinearHostModel> host, bool allow_replicas = true) {
    std::vector<int> devs = device_list();
    if (!allow_replicas || host->shard_world > 1) devs.resize(1);
    auto h = std::make_unique<XLinearHandle>();
    // the engine consumes (and frees) the host arrays while uploading: every replica gets its own copy
    load_replicas(*h, devs, [&](size_t i) { return i ? std::make_unique<pb200::XLinearHostModel>(*host) : std::move(host); });
    return h.release();
}

// rows [0, rows) cut into n contiguous blocks of (nearly) equal nnz (pecos_b200.distributed.split_rows_by_nnz)
std::vector<uint32_t> split_rows_by_nnz(const uint64_t* row_ptr, uint32_t rows, size_t n) {
    std::vector<uint32_t> cut(n + 1, rows);
    cut[0] = 0;
    const uint64_t base = row_ptr[0], total = row_ptr[rows] - base;
    for (size_t i = 1; i < n; ++i) {
        const uint64_t target = base + total * i / n;
        const uint64_t* p = std::lower_bound(row_ptr, row_ptr + rows + 1, target);
        uint32_t r = static_cast<uint32_t>(p - row_ptr);
        if (total == 0) r = static_cast<uint32_t>(static_cast<uint64_t>(rows) * i / n);
        cut[i] = std::max(cut[i - 1], std::min(r, rows));
    }
    return cut;
}

// rows [0, rows) cut into n contiguous blocks of (nearly) equal row counts
std::vector<uint32_t> split_rows_evenly(uint32_t rows, size_t n) {
    std::vector<uint32_t> cut(n + 1);
    for (size_t i = 0; i <= n; ++i) cut[i] = static_cast<uint32_t>(static_cast<uint64_t>(rows) * i / n);
    return cut;
}

// the C-ABI matrix arguments as the engines see them (an absent matrix: empty)
pb200::HostMatrix host_matrix(const ScipyCsrF32* X) {
    return X ? pb200::HostMatrix{X->row_ptr, X->col_idx, X->val, nullptr, X->rows, X->cols} : pb200::HostMatrix{};
}
pb200::HostMatrix host_matrix(const ScipyDrmF32* X) {
    return X ? pb200::HostMatrix{nullptr, nullptr, nullptr, X->val, X->rows, X->cols} : pb200::HostMatrix{};
}

constexpr uint32_t kFanOutMinRows = 256;  // below this many rows per device a single engine serves the call

// Runs fn(i, engine, rows, first row) on contiguous row blocks of x, block i on replica i, one host thread each: blocks of
// (nearly) equal nnz when by_nnz, else of equal row counts.  Returns the number of blocks.
template <typename Engine, typename F>
size_t fan_out_rows(Replicas<Engine>& h, const pb200::HostMatrix& x, bool by_nnz, F&& fn) {
    size_t n = h.engines.size();
    if (static_cast<uint64_t>(x.rows) < static_cast<uint64_t>(kFanOutMinRows) * n) n = 1;
    const auto cut = by_nnz ? split_rows_by_nnz(x.row_ptr, x.rows, n) : split_rows_evenly(x.rows, n);
    fan_out(n, [&](size_t i) { fn(i, *h.engines[i], x.row_block(cut[i], cut[i + 1]), cut[i]); });
    return n;
}

// The shape checks of a query batch against the engine that serves it (MLModel::predict_internal, inference.hpp:2041-2051;
// MLModel::predict_on_selected_outputs, :2148-2158).  A null sel or codes is absent.  Only dense queries are checked for
// their width.
void check_queries(const pb200::XLinearEngine& eng, const pb200::HostMatrix& x, const ScipyCsrF32* sel,
                   const ScipyCsrF32* codes) {
    if (sel && sel->rows != x.rows) throw std::runtime_error("Instance dimension of query and selected output matrix do not match");
    if (codes && codes->rows != x.rows) throw std::runtime_error("Instance dimension of query and prev_layer_pred matrix do not match");
    if (codes && codes->cols != eng.host().nr_codes())  // == C.cols of the one layer
        throw std::runtime_error("Label dimension of prev_layer_pred and C matrix do not match");
    if (x.dense && x.cols != eng.host().nr_features()) throw std::runtime_error("dense query width != nr_features");
}

// Arguments without which a call must not touch a model
const char* required_pp(const char* pp) {
    if (!pp) throw std::runtime_error("single layer: post_processor_str is required");
    return pp;
}
const ScipyCsrF32& required_sel(const ScipyCsrF32* sel) {
    if (!sel) throw std::runtime_error("selected_outputs_csr is required");
    return *sel;
}

// c_xlinear_predict_*: the only XR-Linear call whose rows are split over the replicas (csr by nnz, dense evenly)
void xlinear_predict(XLinearHandle& h, const pb200::HostMatrix& x, uint32_t beam_size, const char* pp, uint32_t only_topk,
                     py_sparse_allocator_t pred_alloc) {
    PB200_LOCK(h)
    check_queries(h.primary(), x, nullptr, nullptr);
    std::vector<pb200::XLinearEngine::Result> parts(h.engines.size());
    const size_t n = fan_out_rows(h, x, x.row_ptr != nullptr, [&](size_t i, pb200::XLinearEngine& eng, const pb200::HostMatrix& rows,
                                                                  uint32_t) { parts[i] = eng.predict(rows, beam_size, pp, only_topk); });
    parts.resize(n);
    emit_results(parts, pred_alloc);
}

// one layer on its primary engine: c_xlinear_single_layer_predict_*, c_mlmodel_predict_*
void layer_predict(XLinearHandle& h, const pb200::HostMatrix& x, const ScipyCsrF32* codes, const char* pp, uint32_t only_topk,
                   py_sparse_allocator_t pred_alloc) {
    PB200_LOCK(h)
    check_queries(h.primary(), x, nullptr, codes);
    emit_result(h.primary().predict_single_layer(x, host_matrix(codes), pp, only_topk), pred_alloc);
}

// scores of exactly the (query, label) pairs of sel on the primary engine: c_xlinear_predict_on_selected_outputs_*,
// c_xlinear_single_layer_predict_on_selected_outputs_*, c_mlmodel_predict_on_selected_outputs_*
void selected_predict(XLinearHandle& h, const pb200::HostMatrix& x, const ScipyCsrF32& sel, const ScipyCsrF32* codes,
                      const char* pp, py_sparse_allocator_t pred_alloc) {
    PB200_LOCK(h)
    check_queries(h.primary(), x, &sel, codes);
    emit_selected(h.primary().predict_selected(x, host_matrix(&sel), pp, host_matrix(codes)), pred_alloc);
}

pb200::DeviceBuffer<unsigned char>* g_flush_buf = nullptr;
std::mutex g_flush_mutex;

}  // namespace

extern "C" {

// ------------------------------------------------ XR-Linear ------------------------------------------------------
void* c_xlinear_load_model_from_disk(const char* model_path) {
    PB200_API_BEGIN
    return make_engine(pb200::load_xlinear_npz_model(model_path, pb200::LT_BINARY_SEARCH_CHUNKED));
    PB200_API_END("c_xlinear_load_model_from_disk")
}

void* c_xlinear_load_model_from_disk_ext(const char* model_path, int weight_matrix_type) {
    PB200_API_BEGIN
    return make_engine(pb200::load_xlinear_npz_model(model_path, weight_matrix_type));
    PB200_API_END("c_xlinear_load_model_from_disk_ext")
}

void* c_xlinear_load_mmap_model_from_disk(const char* model_path, const bool lazy_load) {
    PB200_API_BEGIN
    return make_engine(pb200::load_xlinear_mmap_model(model_path, lazy_load));
    PB200_API_END("c_xlinear_load_mmap_model_from_disk")
}

void c_xlinear_compile_mmap_model(const char* model_path, const char* mmap_model_path) {
    // host-only (no CUDA calls): npz model folder -> the reference's mmap format (libpecos.cpp:133-138)
    PB200_API_BEGIN
    auto host = pb200::load_xlinear_npz_model(model_path, pb200::LT_BINARY_SEARCH_CHUNKED);
    pb200::write_xlinear_mmap_model(*host, mmap_model_path);
    PB200_API_END("c_xlinear_compile_mmap_model")
}

void c_mlmodel_compile_mmap_model(const char* model_path, const char* mmap_model_path) {
    // host-only (no CUDA calls): one npz layer folder -> the reference's single-layer mmap format (libpecos.cpp:32-36)
    PB200_API_BEGIN
    pb200::compile_mlmodel_mmap(model_path, mmap_model_path);
    PB200_API_END("c_mlmodel_compile_mmap_model")
}

void c_xlinear_destruct_model(void* ptr) {
    PB200_API_BEGIN
    delete static_cast<XLinearHandle*>(ptr);
    PB200_API_END("c_xlinear_destruct_model")
}

uint32_t c_xlinear_get_int_attr(void* ptr, const char* attr) {
    PB200_API_BEGIN
    const auto& m = xlinear_of(ptr).primary().host();
    if (std::strcmp(attr, "depth") == 0) return m.depth();
    if (std::strcmp(attr, "nr_features") == 0) return m.nr_features();
    if (std::strcmp(attr, "nr_labels") == 0) return m.nr_labels();
    if (std::strcmp(attr, "nr_codes") == 0) return m.nr_codes();
    throw std::runtime_error(std::string(attr) + " is not implemented in get_int_attr.");
    PB200_API_END("c_xlinear_get_int_attr")
}

int c_xlinear_get_layer_type(void* ptr, int layer_depth) {
    PB200_API_BEGIN
    const auto& m = xlinear_of(ptr).primary().host();
    if (layer_depth < 0 || static_cast<uint32_t>(layer_depth) >= m.depth()) throw std::runtime_error("layer_depth out of range");
    return m.layer_type;
    PB200_API_END("c_xlinear_get_layer_type")
}

}  // extern "C"

namespace {

// Cache of one-layer engines.  The python chain re-sends W and C with every call (pecos/xmc/base.py:934-944), and its
// ctypes shim re-creates the index arrays each time, so pointers of col_ptr / row_idx are useless as identity: the key is
// shape + nnz + value pointer + bias + a content fingerprint over strided samples of all five arrays.
struct LayerKey {
    uint32_t w_rows, w_cols, c_rows, c_cols;
    uint64_t w_nnz, c_nnz;
    const float* w_val;
    uint32_t bias_bits;
    uint64_t fingerprint;
    bool operator==(const LayerKey& o) const {
        return w_rows == o.w_rows && w_cols == o.w_cols && c_rows == o.c_rows && c_cols == o.c_cols && w_nnz == o.w_nnz &&
               c_nnz == o.c_nnz && w_val == o.w_val && bias_bits == o.bias_bits && fingerprint == o.fingerprint;
    }
};

inline uint64_t mix64(uint64_t h, uint64_t v) {
    h ^= v + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
    return h;
}

template <typename T>
uint64_t sample_hash(uint64_t h, const T* a, uint64_t n) {
    if (n == 0) return mix64(h, 0x51ull);
    const uint64_t samples = 4096;
    const uint64_t step = n > samples ? n / samples : 1;
    for (uint64_t i = 0; i < n; i += step) {
        uint64_t v = 0;
        std::memcpy(&v, &a[i], sizeof(T) < 8 ? sizeof(T) : 8);
        h = mix64(h, v + i);
    }
    uint64_t v = 0;
    std::memcpy(&v, &a[n - 1], sizeof(T) < 8 ? sizeof(T) : 8);
    return mix64(h, v);
}

LayerKey make_layer_key(const ScipyCscF32* W, const ScipyCscF32* C, float bias) {
    LayerKey k{};
    k.w_rows = W->rows; k.w_cols = W->cols; k.c_rows = C->rows; k.c_cols = C->cols;
    k.w_nnz = W->col_ptr[W->cols];
    k.c_nnz = C->col_ptr[C->cols];
    k.w_val = W->val;
    std::memcpy(&k.bias_bits, &bias, 4);
    uint64_t h = 0x0123456789ABCDEFull;
    h = sample_hash(h, W->col_ptr, static_cast<uint64_t>(W->cols) + 1);
    h = sample_hash(h, W->row_idx, k.w_nnz);
    h = sample_hash(h, W->val, k.w_nnz);
    h = sample_hash(h, C->col_ptr, static_cast<uint64_t>(C->cols) + 1);
    h = sample_hash(h, C->row_idx, k.c_nnz);
    k.fingerprint = h;
    return k;
}

struct CachedLayer {
    LayerKey key;
    std::shared_ptr<XLinearHandle> handle;
    uint64_t last_use;
};

std::mutex g_layer_cache_mutex;
// heap-allocated and never destroyed: engines must not run CUDA calls from static destructors at process exit
std::vector<CachedLayer>& g_layer_cache = *new std::vector<CachedLayer>();
uint64_t g_layer_clock = 0, g_layer_hits = 0, g_layer_misses = 0;

std::shared_ptr<XLinearHandle> layer_engine(const ScipyCscF32* W, const ScipyCscF32* C, float bias) {
    if (!W || !C) throw std::runtime_error("single layer: W and C are required");
    if (W->cols != C->rows) throw std::runtime_error("single layer: W.cols != C.rows");
    const LayerKey key = make_layer_key(W, C, bias);
    std::lock_guard<std::mutex> lock(g_layer_cache_mutex);
    for (auto& e : g_layer_cache)
        if (e.key == key) { e.last_use = ++g_layer_clock; ++g_layer_hits; return e.handle; }
    ++g_layer_misses;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0)
        throw std::runtime_error("no CUDA device visible: pecos_b200 has no CPU fallback");
    size_t cap = 8;
    if (const char* env = std::getenv("PB200_LAYER_CACHE")) cap = static_cast<size_t>(std::max(1, std::atoi(env)));
    while (g_layer_cache.size() >= cap) {  // evict the least recently used engine (frees its HBM once callers are done)
        size_t victim = 0;
        for (size_t i = 1; i < g_layer_cache.size(); ++i)
            if (g_layer_cache[i].last_use < g_layer_cache[victim].last_use) victim = i;
        g_layer_cache.erase(g_layer_cache.begin() + static_cast<std::ptrdiff_t>(victim));
    }
    const pb200::CscRaw w{W->rows, W->cols, W->col_ptr, W->row_idx, W->val};
    const pb200::CscRaw c{C->rows, C->cols, C->col_ptr, C->row_idx, C->val};
    auto h = std::make_shared<XLinearHandle>();
    h->engines.push_back(std::make_unique<pb200::XLinearEngine>(pb200::make_single_layer_model(w, c, bias), g_device.load()));
    g_layer_cache.push_back(CachedLayer{key, h, ++g_layer_clock});
    return h;
}

}  // namespace

extern "C" {

// The six XR-Linear predict operations of one query type (libpecos.cpp:52-113, :158-274).  Single layers are the python
// chain's (pecos/xmc/base.py:934-944): their engine comes from the layer cache, and post_processor_str and
// selected_outputs_csr are checked before any layer is uploaded.  only_topk 0: the mlmodel calls use the stored value
// (inference.hpp:2055); a single layer passes it on and returns empty rows (inference.hpp:1237).
#define PB200_XLINEAR_API(SUFFIX, MAT_T)                                                                                      \
    void c_xlinear_predict##SUFFIX(void* ptr, const MAT_T* X, const uint32_t overridden_beam_size,                           \
                                   const char* overridden_post_processor_str, const uint32_t overridden_only_topk,           \
                                   const int threads, py_sparse_allocator_t pred_alloc) {                                    \
        (void)threads;                                                                                                       \
        PB200_API_BEGIN                                                                                                      \
        xlinear_predict(xlinear_of(ptr), host_matrix(X), overridden_beam_size, overridden_post_processor_str,               \
                        overridden_only_topk, pred_alloc);                                                                   \
        PB200_API_END("c_xlinear_predict" #SUFFIX)                                                                           \
    }                                                                                                                        \
    void c_xlinear_predict_on_selected_outputs##SUFFIX(void* ptr, const MAT_T* X, const ScipyCsrF32* selected_outputs_csr,  \
                                                       const char* overridden_post_processor_str, const int threads,         \
                                                       py_sparse_allocator_t pred_alloc) {                                   \
        (void)threads;                                                                                                       \
        PB200_API_BEGIN                                                                                                      \
        auto& h = xlinear_of(ptr);                                                                                           \
        selected_predict(h, host_matrix(X), required_sel(selected_outputs_csr), nullptr, overridden_post_processor_str,     \
                         pred_alloc);                                                                                        \
        PB200_API_END("c_xlinear_predict_on_selected_outputs" #SUFFIX)                                                       \
    }                                                                                                                        \
    void c_xlinear_single_layer_predict##SUFFIX(const MAT_T* input_x, const ScipyCsrF32* csr_codes, ScipyCscF32* W,         \
                                                ScipyCscF32* C, const char* post_processor_str, const uint32_t only_topk,    \
                                                const int num_threads, const float bias, py_sparse_allocator_t pred_alloc) { \
        (void)num_threads;                                                                                                   \
        PB200_API_BEGIN                                                                                                      \
        const char* pp = required_pp(post_processor_str);                                                                    \
        layer_predict(*layer_engine(W, C, bias), host_matrix(input_x), csr_codes, pp, only_topk, pred_alloc);               \
        PB200_API_END("c_xlinear_single_layer_predict" #SUFFIX)                                                              \
    }                                                                                                                        \
    void c_xlinear_single_layer_predict_on_selected_outputs##SUFFIX(                                                         \
        const MAT_T* input_x, const ScipyCsrF32* selected_outputs_csr, const ScipyCsrF32* csr_codes, ScipyCscF32* W,        \
        ScipyCscF32* C, const char* post_processor_str, const int num_threads, const float bias,                             \
        py_sparse_allocator_t pred_alloc) {                                                                                  \
        (void)num_threads;                                                                                                   \
        PB200_API_BEGIN                                                                                                      \
        const char* pp = required_pp(post_processor_str);                                                                    \
        const ScipyCsrF32& sel = required_sel(selected_outputs_csr);                                                         \
        selected_predict(*layer_engine(W, C, bias), host_matrix(input_x), sel, csr_codes, pp, pred_alloc);                  \
        PB200_API_END("c_xlinear_single_layer_predict_on_selected_outputs" #SUFFIX)                                          \
    }                                                                                                                        \
    void c_mlmodel_predict##SUFFIX(void* ptr, const MAT_T* input_x, const ScipyCsrF32* csr_codes,                           \
                                   const char* overridden_post_processor, const uint32_t overridden_only_topk,               \
                                   const int num_threads, py_sparse_allocator_t pred_alloc) {                                \
        (void)num_threads;                                                                                                   \
        PB200_API_BEGIN                                                                                                      \
        auto& h = xlinear_of(ptr);                                                                                           \
        const uint32_t k = overridden_only_topk > 0 ? overridden_only_topk                                                   \
                                                    : static_cast<uint32_t>(h.primary().host().layers.at(0).only_topk);      \
        layer_predict(h, host_matrix(input_x), csr_codes, overridden_post_processor, k, pred_alloc);                        \
        PB200_API_END("c_mlmodel_predict" #SUFFIX)                                                                           \
    }                                                                                                                        \
    void c_mlmodel_predict_on_selected_outputs##SUFFIX(void* ptr, const MAT_T* input_x,                                      \
                                                       const ScipyCsrF32* selected_outputs_csr, const ScipyCsrF32* csr_codes, \
                                                       const char* overridden_post_processor, const int num_threads,         \
                                                       py_sparse_allocator_t pred_alloc) {                                   \
        (void)num_threads;                                                                                                   \
        PB200_API_BEGIN                                                                                                      \
        auto& h = xlinear_of(ptr);                                                                                           \
        selected_predict(h, host_matrix(input_x), required_sel(selected_outputs_csr), csr_codes, overridden_post_processor, \
                         pred_alloc);                                                                                        \
        PB200_API_END("c_mlmodel_predict_on_selected_outputs" #SUFFIX)                                                       \
    }

PB200_XLINEAR_API(_csr_f32, ScipyCsrF32)
PB200_XLINEAR_API(_drm_f32, ScipyDrmF32)

uint32_t pb200_layer_cache_clear(void) {
    PB200_API_BEGIN
    std::lock_guard<std::mutex> lock(g_layer_cache_mutex);
    const uint32_t n = static_cast<uint32_t>(g_layer_cache.size());
    g_layer_cache.clear();
    return n;
    PB200_API_END("pb200_layer_cache_clear")
}

void pb200_layer_cache_info(uint64_t* out) {
    PB200_API_BEGIN
    std::lock_guard<std::mutex> lock(g_layer_cache_mutex);
    out[0] = g_layer_cache.size(); out[1] = g_layer_hits; out[2] = g_layer_misses;
    PB200_API_END("pb200_layer_cache_info")
}

// ------------------------------------------------ single-layer mmap handles (c_mlmodel_*) -------------------------
// pecos/core/libpecos.cpp:37-113: MLModel<csc_t> saved by save_mmap, served here by a one-layer engine.
void* c_mlmodel_load_mmap_model(const char* model_path, const bool lazy_load) {
    PB200_API_BEGIN
    return make_engine(pb200::load_mlmodel_mmap(model_path, lazy_load), false);
    PB200_API_END("c_mlmodel_load_mmap_model")
}

void c_mlmodel_destruct_model(void* ptr) {
    PB200_API_BEGIN
    delete static_cast<XLinearHandle*>(ptr);
    PB200_API_END("c_mlmodel_destruct_model")
}

uint32_t c_mlmodel_get_int_attr(void* ptr, const char* attr) {
    PB200_API_BEGIN
    const auto& m = xlinear_of(ptr).primary().host();
    // MLModel<csc_t>::label_count() = W.cols: the csc layout is never rearranged, so pruned / permuted trees report every
    // column of W (our chunked layout scores nnz(C) columns; out_cols keeps the reference's count)
    if (std::strcmp(attr, "nr_labels") == 0) return m.layers.back().out_cols;
    if (std::strcmp(attr, "nr_codes") == 0) return m.nr_codes();
    if (std::strcmp(attr, "nr_features") == 0) return m.nr_features();
    throw std::runtime_error(std::string(attr) + " is not implemented in get_int_attr.");
    PB200_API_END("c_mlmodel_get_int_attr")
}

// ------------------------------------------------ additions ------------------------------------------------------
const char* pb200_version(void) { return "pecos_b200 0.1 (sm_90a)"; }

int pb200_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

int pb200_set_device(int device) {
    int n = pb200_device_count();
    if (device < 0 || device >= n) return 1;
    g_device.store(device);
    return cudaSetDevice(device) == cudaSuccess ? 0 : 1;
}

int pb200_get_device(void) { return g_device.load(); }

void* pb200_host_alloc(size_t bytes) {
    PB200_API_BEGIN
    void* p = nullptr;
    PB200_CUDA(cudaSetDevice(g_device.load()));
    PB200_CUDA(cudaMallocHost(&p, bytes ? bytes : 1));
    return p;
    PB200_API_END("pb200_host_alloc")
}

void pb200_host_free(void* ptr) {
    if (ptr) cudaFreeHost(ptr);
}

void pb200_l2_flush(void) {
    PB200_API_BEGIN
    std::lock_guard<std::mutex> lock(g_flush_mutex);
    PB200_CUDA(cudaSetDevice(g_device.load()));
    if (!g_flush_buf) g_flush_buf = new pb200::DeviceBuffer<unsigned char>();
    const uint64_t bytes = 512ull << 20;  // 10x the 50 MB L2 of an H100
    g_flush_buf->reserve(bytes);
    static int tick = 0;
    PB200_CUDA(cudaMemset(g_flush_buf->get(), (++tick) & 0xFF, bytes));
    PB200_CUDA(cudaDeviceSynchronize());
    PB200_API_END("pb200_l2_flush")
}

// ------------------------------------------------ index construction (sparse HNSW builder) ----------------------------
void pb200_sparse_block_distances(int device, int metric, const void* row_ptr, const void* ent, const void* q_ids, uint32_t nq,
                                  const void* col_ptr, const void* post, uint32_t c0, uint32_t nc, void* out, void* work,
                                  void* stream) {
    PB200_API_BEGIN
    pb200::sparse_block_distances(device, metric, static_cast<const uint64_t*>(row_ptr), static_cast<const uint2*>(ent),
                                  static_cast<const int64_t*>(q_ids), nq, static_cast<const uint64_t*>(col_ptr),
                                  static_cast<const uint2*>(post), c0, nc, static_cast<float*>(out),
                                  static_cast<unsigned long long*>(work), static_cast<cudaStream_t>(stream));
    PB200_API_END("pb200_sparse_block_distances")
}

void pb200_sparse_candidate_distances(int device, int metric, const void* row_ptr, const void* ent, const void* cand, uint32_t n,
                                      uint32_t C, void* out, void* work, void* stream) {
    PB200_API_BEGIN
    pb200::sparse_candidate_distances(device, metric, static_cast<const uint64_t*>(row_ptr), static_cast<const uint2*>(ent),
                                      static_cast<const int64_t*>(cand), n, C, static_cast<float*>(out),
                                      static_cast<unsigned long long*>(work), static_cast<cudaStream_t>(stream));
    PB200_API_END("pb200_sparse_candidate_distances")
}

void pb200_xlinear_resident_upload_csr(void* ptr, const ScipyCsrF32* X) {
    PB200_API_BEGIN
    PB200_LOCK(xlinear_of(ptr))
    xlinear_of(ptr).primary().resident_upload_csr(host_matrix(X));
    PB200_API_END("pb200_xlinear_resident_upload_csr")
}

double pb200_xlinear_resident_predict(void* ptr, uint32_t beam, const char* pp, uint32_t topk, int collect_stats) {
    PB200_API_BEGIN
    PB200_LOCK(xlinear_of(ptr))
    return xlinear_of(ptr).primary().resident_predict(beam, pp, topk, collect_stats != 0);
    PB200_API_END("pb200_xlinear_resident_predict")
}

void pb200_xlinear_resident_fetch(void* ptr, py_sparse_allocator_t pred_alloc) {
    PB200_API_BEGIN
    PB200_LOCK(xlinear_of(ptr))
    emit_result(xlinear_of(ptr).primary().resident_fetch(), pred_alloc);
    PB200_API_END("pb200_xlinear_resident_fetch")
}

void* pb200_xlinear_load_sharded(const char* model_path, int weight_matrix_type, uint32_t shard_rank, uint32_t shard_world) {
    PB200_API_BEGIN
    if (weight_matrix_type < 0) return make_engine(pb200::load_xlinear_mmap_model(model_path, false, shard_rank, shard_world), false);
    return make_engine(pb200::load_xlinear_npz_model(model_path, weight_matrix_type, shard_rank, shard_world), false);
    PB200_API_END("pb200_xlinear_load_sharded")
}

void pb200_xlinear_get_shard(void* ptr, uint32_t* out) {
    PB200_API_BEGIN
    const auto& m = xlinear_of(ptr).primary().host();
    out[0] = m.shard_rank; out[1] = m.shard_world; out[2] = m.leaf_chunk_begin; out[3] = m.leaf_chunk_end;
    PB200_API_END("pb200_xlinear_get_shard")
}

uint32_t pb200_xlinear_sharded_local_csr_packed(void* ptr, const ScipyCsrF32* X, uint32_t beam, const char* pp, uint32_t topk,
                                                uint32_t stride_capacity, void* rec_dev) {
    PB200_API_BEGIN
    PB200_LOCK(xlinear_of(ptr))
    return xlinear_of(ptr).primary().sharded_local_csr_packed(host_matrix(X), beam, pp, topk, stride_capacity, rec_dev);
    PB200_API_END("pb200_xlinear_sharded_local_csr_packed")
}

void pb200_xlinear_sharded_merge_packed(void* ptr, uint32_t world, uint32_t rows, uint32_t stride, uint32_t topk, const void* g_rec,
                                        py_sparse_allocator_t pred_alloc) {
    PB200_API_BEGIN
    PB200_LOCK(xlinear_of(ptr))
    emit_result(xlinear_of(ptr).primary().sharded_merge_packed(world, rows, stride, topk, g_rec), pred_alloc);
    PB200_API_END("pb200_xlinear_sharded_merge_packed")
}

void pb200_xlinear_set_profile(void* ptr, int on) {
    PB200_API_BEGIN
    PB200_LOCK(xlinear_of(ptr))
    xlinear_of(ptr).primary().set_profile(on != 0);
    PB200_API_END("pb200_xlinear_set_profile")
}

int pb200_xlinear_set_lookup(void* ptr, int on) {
    PB200_API_BEGIN
    PB200_LOCK(xlinear_of(ptr))
    xlinear_of(ptr).primary().set_kernel_mode(on);
    return xlinear_of(ptr).primary().has_feature_maps() ? 1 : 0;
    PB200_API_END("pb200_xlinear_set_lookup")
}

void pb200_xlinear_reset_profile(void* ptr) {
    PB200_API_BEGIN
    PB200_LOCK(xlinear_of(ptr))
    xlinear_of(ptr).primary().reset_profile();
    PB200_API_END("pb200_xlinear_reset_profile")
}

void pb200_xlinear_get_profile(void* ptr, double* out) {
    PB200_API_BEGIN
    PB200_LOCK(xlinear_of(ptr))
    const auto& p = xlinear_of(ptr).primary().layer_profile();
    for (size_t d = 0; d < p.size(); ++d) { out[2 * d] = p[d].scores_ms; out[2 * d + 1] = p[d].topk_ms; }
    PB200_API_END("pb200_xlinear_get_profile")
}

void pb200_xlinear_get_kernel_ids(void* ptr, int* out) {
    PB200_API_BEGIN
    PB200_LOCK(xlinear_of(ptr))
    const auto& p = xlinear_of(ptr).primary().layer_profile();
    for (size_t d = 0; d < p.size(); ++d) { out[2 * d] = p[d].scores_kernel; out[2 * d + 1] = p[d].topk_kernel; }
    PB200_API_END("pb200_xlinear_get_kernel_ids")
}

int pb200_xlinear_cm_info(void* ptr, int layer, uint64_t* out) {
    PB200_API_BEGIN
    PB200_LOCK(xlinear_of(ptr))
    const pb200::CmShape* s = xlinear_of(ptr).primary().cm_shape_of(layer);
    if (!s) return 1;
    out[0] = s->ok ? 1 : 0; out[1] = s->direct ? 1 : 0; out[2] = s->col_cap; out[3] = s->n_vc; out[4] = s->img_bytes;
    out[5] = s->warps_fit;
    return 0;
    PB200_API_END("pb200_xlinear_cm_info")
}

uint32_t pb200_xlinear_beam_limit(int topk) { return topk ? pb200::kXlBeamMaxTopk : pb200::kXlBeamMax; }

void pb200_xlinear_get_stats(void* ptr, uint64_t* out) {
    PB200_API_BEGIN
    PB200_LOCK(xlinear_of(ptr))
    const auto& s = xlinear_of(ptr).primary().layer_stats();
    for (size_t d = 0; d < s.size(); ++d) {
        out[7 * d + 0] = s[d].chunks; out[7 * d + 1] = s[d].chunk_rows; out[7 * d + 2] = s[d].matched;
        out[7 * d + 3] = s[d].entries; out[7 * d + 4] = s[d].out_cols; out[7 * d + 5] = s[d].query_nnz;
        out[7 * d + 6] = s[d].beam_out;
    }
    PB200_API_END("pb200_xlinear_get_stats")
}

uint64_t pb200_xlinear_launches(void* ptr) {
    PB200_API_BEGIN
    return xlinear_of(ptr).primary().launches();
    PB200_API_END("pb200_xlinear_launches")
}

uint32_t pb200_xlinear_replicas(void* ptr) {
    PB200_API_BEGIN
    return static_cast<uint32_t>(xlinear_of(ptr).engines.size());
    PB200_API_END("pb200_xlinear_replicas")
}

uint64_t pb200_xlinear_model_bytes(void* ptr) {
    PB200_API_BEGIN
    return xlinear_of(ptr).primary().model_bytes();
    PB200_API_END("pb200_xlinear_model_bytes")
}

// host-only inspection (no CUDA calls)
void* pb200_xlinear_host_load(const char* model_path, int kind) {
    PB200_API_BEGIN
    std::unique_ptr<pb200::XLinearHostModel> m =
        kind == 1 ? pb200::load_xlinear_mmap_model(model_path, false)
                  : pb200::load_xlinear_npz_model(model_path, pb200::LT_BINARY_SEARCH_CHUNKED);
    return m.release();
    PB200_API_END("pb200_xlinear_host_load")
}

void* pb200_xlinear_host_from_csc(const ScipyCscF32* W, const ScipyCscF32* C, float bias) {
    PB200_API_BEGIN
    const pb200::CscRaw w{W->rows, W->cols, W->col_ptr, W->row_idx, W->val};
    const pb200::CscRaw c{C->rows, C->cols, C->col_ptr, C->row_idx, C->val};
    return pb200::make_single_layer_model(w, c, bias).release();
    PB200_API_END("pb200_xlinear_host_from_csc")
}

void* pb200_xlinear_host_prefix_layer(void* hptr) {
    PB200_API_BEGIN
    const auto& H = *static_cast<pb200::XLinearHostModel*>(hptr);
    if (H.depth() < 2) throw std::runtime_error("pecos_b200: the prefix layer needs a model of depth >= 2");
    auto m = std::make_unique<pb200::XLinearHostModel>();
    m->layers.resize(1);
    pb200::build_prefix_layer(H.layers[0], H.layers[1], m->layers[0]);
    return m.release();
    PB200_API_END("pb200_xlinear_host_prefix_layer")
}

void pb200_xlinear_host_free(void* hptr) { delete static_cast<pb200::XLinearHostModel*>(hptr); }

int pb200_xlinear_host_plan_fits(void* hptr, uint32_t beam_size, uint32_t only_topk, uint32_t* out) {
    PB200_API_BEGIN
    if (!hptr) throw std::runtime_error("null host model");
    return plan_fits(*static_cast<pb200::XLinearHostModel*>(hptr), beam_size, only_topk, out);
    PB200_API_END("pb200_xlinear_host_plan_fits")
}

int pb200_xlinear_plan_fits(void* ptr, uint32_t beam_size, uint32_t only_topk, uint32_t* out) {
    PB200_API_BEGIN
    // host model only: callable while the device is busy
    return plan_fits(xlinear_of(ptr).primary().host(), beam_size, only_topk, out);
    PB200_API_END("pb200_xlinear_plan_fits")
}

uint32_t pb200_xlinear_plan_stride(void* ptr, int host, uint32_t beam_size, uint32_t only_topk) {
    PB200_API_BEGIN
    if (!ptr) throw std::runtime_error("null model handle");
    // host model only: callable while the device is busy
    const pb200::XLinearHostModel& m = host ? *static_cast<pb200::XLinearHostModel*>(ptr) : xlinear_of(ptr).primary().host();
    return pb200::xlinear_plan_stride(m, beam_size, only_topk);
    PB200_API_END("pb200_xlinear_plan_stride")
}

uint32_t pb200_xlinear_host_depth(void* hptr) { return static_cast<pb200::XLinearHostModel*>(hptr)->depth(); }

void pb200_xlinear_host_layer_dims(void* hptr, uint32_t layer, uint64_t* out) {
    PB200_API_BEGIN
    const auto& L = static_cast<pb200::XLinearHostModel*>(hptr)->layers.at(layer);
    out[0] = L.w_rows; out[1] = L.n_cols; out[2] = L.out_cols; out[3] = L.n_chunks; out[4] = L.c_max;
    out[5] = L.meta.size(); out[6] = L.entries.size(); out[7] = L.label_of_col.size();
    PB200_API_END("pb200_xlinear_host_layer_dims")
}

void pb200_xlinear_host_layer_export(void* hptr, uint32_t layer, void* chunks32, uint32_t* meta, void* entries8,
                                     uint32_t* label_of_col) {
    PB200_API_BEGIN
    const auto& L = static_cast<pb200::XLinearHostModel*>(hptr)->layers.at(layer);
    if (chunks32) std::memcpy(chunks32, L.chunks.data(), L.chunks.size() * sizeof(pb200::ChunkHeader));
    if (meta) std::memcpy(meta, L.meta.data(), L.meta.size() * 4);
    if (entries8) std::memcpy(entries8, L.entries.data(), L.entries.size() * 8);
    if (label_of_col) std::memcpy(label_of_col, L.label_of_col.data(), L.label_of_col.size() * 4);
    PB200_API_END("pb200_xlinear_host_layer_export")
}

}  // extern "C"

// ------------------------------------------------ HNSW ----------------------------------------------------------
namespace {

struct HnswSearchers {  // the reference hands out a vector<Searcher>; our scratch lives with the engine (per warp)
    HnswHandle* owner;
    uint32_t num_searcher;
};

void* hnsw_load(const char* model_dir, bool lazy_load, int metric, bool sparse) {
    auto h = std::make_unique<HnswHandle>();
    // the host index is a view of the memory-mapped file: every replica maps it again (shared page cache)
    load_replicas(*h, device_list(), [&](size_t) { return pb200::load_hnsw_index(model_dir, metric, lazy_load, sparse); });
    h->model_dir = model_dir;
    return h.release();
}

// replicas: even row blocks, each engine writes its slice of the caller's arrays
void hnsw_predict(void* model_ptr, const pb200::HostMatrix& x, uint32_t* ret_idx, float* ret_val, uint32_t efS, uint32_t topk,
                  int metric) {
    auto& h = hnsw_of(model_ptr);
    PB200_LOCK(h)
    if (h.primary().metric() != metric) throw std::runtime_error("HNSW handle was loaded with a different metric");
    fan_out_rows(h, x, false, [&](size_t, pb200::HnswEngine& eng, const pb200::HostMatrix& rows, uint32_t r0) {
        const uint64_t o = static_cast<uint64_t>(r0) * topk;
        eng.predict(rows, efS, topk, ret_idx + o, ret_val + o);
    });
}

}  // namespace

extern "C" {

// Handles are library-specific.  Indices TRAINED by the reference (c_ann_hnsw_train_* stays on the reference library) are
// reference handles, yet once the overlay has re-pointed destruct / predict / searchers_* / save at this library the reference's
// Python hands them to us.  Live handles and searcher tokens created HERE are therefore registered; anything else is forwarded
// to the reference's own function, which the overlay registers through pb200_hnsw_set_foreign (without it: a clear fatal error
// instead of undefined behaviour).
typedef void (*hnsw_destruct_fn)(void*);
typedef void* (*hnsw_searchers_create_fn)(void*, uint32_t);
typedef void (*hnsw_predict_fn)(void*, const void*, uint32_t*, float*, uint32_t, uint32_t, int32_t, void*);
typedef void (*hnsw_save_fn)(void*, const char*);
struct HnswForeign {
    hnsw_destruct_fn destruct = nullptr;
    hnsw_searchers_create_fn searchers_create = nullptr;
    hnsw_destruct_fn searchers_destruct = nullptr;
    hnsw_predict_fn predict = nullptr;
    hnsw_save_fn save = nullptr;
};
}  // extern "C"

namespace {
std::mutex g_hnsw_reg_mutex;
std::unordered_set<void*>& g_hnsw_models = *new std::unordered_set<void*>();
std::unordered_set<void*>& g_hnsw_tokens = *new std::unordered_set<void*>();
HnswForeign g_hnsw_foreign[4];  // [metric + 2 * sparse]

bool hnsw_is_ours(void* p, bool token = false) {
    std::lock_guard<std::mutex> lock(g_hnsw_reg_mutex);
    return (token ? g_hnsw_tokens : g_hnsw_models).count(p) != 0;
}
void hnsw_register(void* p, bool token, bool add) {
    std::lock_guard<std::mutex> lock(g_hnsw_reg_mutex);
    auto& s = token ? g_hnsw_tokens : g_hnsw_models;
    if (add) s.insert(p); else s.erase(p);
}
[[noreturn]] void hnsw_foreign_missing(const char* what) {
    throw std::runtime_error(std::string(what) + ": the handle was not created by pecos_b200 (an index trained by the reference "
                             "library?) and no reference functions were registered with pb200_hnsw_set_foreign");
}
void hnsw_save_copy(void* model_ptr, const char* model_dir) {
    // an index loaded here is a view of <dir>/index.mmap_store + config.json written by the reference: saving = copying them
    const std::string src = static_cast<HnswHandle*>(model_ptr)->model_dir, dst(model_dir);
    if (system(("mkdir -p '" + dst + "'").c_str()) != 0) throw std::runtime_error("cannot create " + dst);
    for (const char* f : {"/config.json", "/index.mmap_store"}) {
        std::FILE* in = std::fopen((src + f).c_str(), "rb");
        if (!in) throw std::runtime_error("cannot read " + src + f);
        std::FILE* out = std::fopen((dst + f).c_str(), "wb");
        if (!out) { std::fclose(in); throw std::runtime_error("cannot write " + dst + f); }
        std::vector<char> buf(1 << 20);
        size_t n;
        while ((n = std::fread(buf.data(), 1, buf.size(), in)) > 0) std::fwrite(buf.data(), 1, n, out);
        std::fclose(in);
        std::fclose(out);
    }
}
}  // namespace

extern "C" {

void pb200_hnsw_set_foreign(int metric, void* destruct, void* searchers_create, void* searchers_destruct, void* predict, void* save) {
    if (metric < 0 || metric > 3) return;  // 0 / 1: dense ip / l2; 2 / 3: sparse (csr) ip / l2
    HnswForeign& f = g_hnsw_foreign[metric];
    f.destruct = reinterpret_cast<hnsw_destruct_fn>(destruct);
    f.searchers_create = reinterpret_cast<hnsw_searchers_create_fn>(searchers_create);
    f.searchers_destruct = reinterpret_cast<hnsw_destruct_fn>(searchers_destruct);
    f.predict = reinterpret_cast<hnsw_predict_fn>(predict);
    f.save = reinterpret_cast<hnsw_save_fn>(save);
}

#define PB200_HNSW_API(SUFFIX, METRIC, MAT_T, SPARSE)                                                                              \
    void* c_ann_hnsw_load##SUFFIX(const char* model_dir, const bool lazy_load) {                                        \
        PB200_API_BEGIN                                                                                                 \
        void* h = hnsw_load(model_dir, lazy_load, METRIC, SPARSE);                                                              \
        hnsw_register(h, false, true);                                                                                  \
        return h;                                                                                                       \
        PB200_API_END("c_ann_hnsw_load" #SUFFIX)                                                                        \
    }                                                                                                                   \
    void c_ann_hnsw_destruct##SUFFIX(void* model_ptr) {                                                                 \
        PB200_API_BEGIN                                                                                                 \
        if (!model_ptr) return;                                                                                         \
        if (!hnsw_is_ours(model_ptr)) {                                                                                 \
            if (!g_hnsw_foreign[METRIC + 2 * SPARSE].destruct) hnsw_foreign_missing("c_ann_hnsw_destruct" #SUFFIX);                  \
            g_hnsw_foreign[METRIC + 2 * SPARSE].destruct(model_ptr);                                                                 \
            return;                                                                                                     \
        }                                                                                                               \
        hnsw_register(model_ptr, false, false);                                                                         \
        delete static_cast<HnswHandle*>(model_ptr);                                                                     \
        PB200_API_END("c_ann_hnsw_destruct" #SUFFIX)                                                                    \
    }                                                                                                                   \
    void* c_ann_hnsw_searchers_create##SUFFIX(void* model_ptr, uint32_t num_searcher) {                                 \
        PB200_API_BEGIN                                                                                                 \
        if (!hnsw_is_ours(model_ptr)) {                                                                                 \
            if (!g_hnsw_foreign[METRIC + 2 * SPARSE].searchers_create) hnsw_foreign_missing("c_ann_hnsw_searchers_create" #SUFFIX);  \
            return g_hnsw_foreign[METRIC + 2 * SPARSE].searchers_create(model_ptr, num_searcher);                                    \
        }                                                                                                               \
        void* t = new HnswSearchers{static_cast<HnswHandle*>(model_ptr), num_searcher};                                 \
        hnsw_register(t, true, true);                                                                                   \
        return t;                                                                                                       \
        PB200_API_END("c_ann_hnsw_searchers_create" #SUFFIX)                                                            \
    }                                                                                                                   \
    void c_ann_hnsw_searchers_destruct##SUFFIX(void* searchers_ptr) {                                                   \
        PB200_API_BEGIN                                                                                                 \
        if (!searchers_ptr) return;                                                                                     \
        if (!hnsw_is_ours(searchers_ptr, true)) {                                                                       \
            if (!g_hnsw_foreign[METRIC + 2 * SPARSE].searchers_destruct) hnsw_foreign_missing("c_ann_hnsw_searchers_destruct" #SUFFIX); \
            g_hnsw_foreign[METRIC + 2 * SPARSE].searchers_destruct(searchers_ptr);                                                   \
            return;                                                                                                     \
        }                                                                                                               \
        hnsw_register(searchers_ptr, true, false);                                                                      \
        delete static_cast<HnswSearchers*>(searchers_ptr);                                                              \
        PB200_API_END("c_ann_hnsw_searchers_destruct" #SUFFIX)                                                          \
    }                                                                                                                   \
    void c_ann_hnsw_predict##SUFFIX(void* model_ptr, const MAT_T* pX, uint32_t* ret_idx, float* ret_val,                \
                                    uint32_t efS, uint32_t topk, int32_t threads, void* searchers_ptr) {                \
        PB200_API_BEGIN                                                                                                 \
        if (!hnsw_is_ours(model_ptr)) {                                                                                 \
            if (!g_hnsw_foreign[METRIC + 2 * SPARSE].predict) hnsw_foreign_missing("c_ann_hnsw_predict" #SUFFIX);                    \
            g_hnsw_foreign[METRIC + 2 * SPARSE].predict(model_ptr, pX, ret_idx, ret_val, efS, topk, threads, searchers_ptr);         \
            return;                                                                                                     \
        }                                                                                                               \
        hnsw_predict(model_ptr, host_matrix(pX), ret_idx, ret_val, efS, topk, METRIC);                                  \
        PB200_API_END("c_ann_hnsw_predict" #SUFFIX)                                                                     \
    }                                                                                                                   \
    void c_ann_hnsw_save##SUFFIX(void* model_ptr, const char* model_dir) {                                              \
        PB200_API_BEGIN                                                                                                 \
        if (!hnsw_is_ours(model_ptr)) {                                                                                 \
            if (!g_hnsw_foreign[METRIC + 2 * SPARSE].save) hnsw_foreign_missing("c_ann_hnsw_save" #SUFFIX);                          \
            g_hnsw_foreign[METRIC + 2 * SPARSE].save(model_ptr, model_dir);                                                          \
            return;                                                                                                     \
        }                                                                                                               \
        hnsw_save_copy(model_ptr, model_dir);                                                                           \
        PB200_API_END("c_ann_hnsw_save" #SUFFIX)                                                                        \
    }

PB200_HNSW_API(_drm_ip_f32, pb200::HNSW_IP, ScipyDrmF32, 0)
PB200_HNSW_API(_drm_l2_f32, pb200::HNSW_L2, ScipyDrmF32, 0)
PB200_HNSW_API(_csr_ip_f32, pb200::HNSW_IP, ScipyCsrF32, 1)
PB200_HNSW_API(_csr_l2_f32, pb200::HNSW_L2, ScipyCsrF32, 1)

void pb200_hnsw_resident_upload_csr(void* model_ptr, const ScipyCsrF32* pX) {
    PB200_API_BEGIN
    PB200_LOCK(hnsw_of(model_ptr))
    hnsw_of(model_ptr).primary().resident_upload(host_matrix(pX));
    PB200_API_END("pb200_hnsw_resident_upload_csr")
}

void pb200_hnsw_resident_upload(void* model_ptr, const ScipyDrmF32* pX) {
    PB200_API_BEGIN
    PB200_LOCK(hnsw_of(model_ptr))
    hnsw_of(model_ptr).primary().resident_upload(host_matrix(pX));
    PB200_API_END("pb200_hnsw_resident_upload")
}

double pb200_hnsw_resident_predict(void* model_ptr, uint32_t efS, uint32_t topk) {
    PB200_API_BEGIN
    PB200_LOCK(hnsw_of(model_ptr))
    return hnsw_of(model_ptr).primary().resident_predict(efS, topk);
    PB200_API_END("pb200_hnsw_resident_predict")
}

void pb200_hnsw_resident_fetch(void* model_ptr, uint32_t* ret_idx, float* ret_val) {
    PB200_API_BEGIN
    PB200_LOCK(hnsw_of(model_ptr))
    hnsw_of(model_ptr).primary().resident_fetch(ret_idx, ret_val);
    PB200_API_END("pb200_hnsw_resident_fetch")
}

// index sharding: the handle's primary engine holds one shard (PB200_DEVICES replicas are not used)
void pb200_hnsw_sharded_local_packed_drm(void* model_ptr, const ScipyDrmF32* pX, uint32_t efS, uint32_t topk, uint32_t rank,
                                         uint32_t id_offset, void* rec_dev) {
    PB200_API_BEGIN
    PB200_LOCK(hnsw_of(model_ptr))
    hnsw_of(model_ptr).primary().sharded_local_packed(host_matrix(pX), efS, topk, rank, id_offset, rec_dev);
    PB200_API_END("pb200_hnsw_sharded_local_packed_drm")
}

void pb200_hnsw_sharded_local_packed_csr(void* model_ptr, const ScipyCsrF32* pX, uint32_t efS, uint32_t topk, uint32_t rank,
                                         uint32_t id_offset, void* rec_dev) {
    PB200_API_BEGIN
    PB200_LOCK(hnsw_of(model_ptr))
    hnsw_of(model_ptr).primary().sharded_local_packed(host_matrix(pX), efS, topk, rank, id_offset, rec_dev);
    PB200_API_END("pb200_hnsw_sharded_local_packed_csr")
}

void pb200_hnsw_sharded_merge_packed(void* model_ptr, uint32_t world, uint32_t rows, uint32_t topk, const void* g_rec,
                                     uint32_t* ret_idx, float* ret_val) {
    PB200_API_BEGIN
    PB200_LOCK(hnsw_of(model_ptr))
    hnsw_of(model_ptr).primary().sharded_merge_packed(world, rows, topk, g_rec, ret_idx, ret_val);
    PB200_API_END("pb200_hnsw_sharded_merge_packed")
}

int pb200_hnsw_set_stages(void* model_ptr, int stages) {
    PB200_API_BEGIN
    PB200_LOCK(hnsw_of(model_ptr))
    hnsw_of(model_ptr).primary().set_stages(stages);
    return hnsw_of(model_ptr).primary().stages();
    PB200_API_END("pb200_hnsw_set_stages")
}

void pb200_hnsw_launch_info(void* model_ptr, uint64_t* out) {
    PB200_API_BEGIN
    PB200_LOCK(hnsw_of(model_ptr))
    hnsw_of(model_ptr).primary().launch_info(out);
    PB200_API_END("pb200_hnsw_launch_info")
}

// Host-only: whether a search (efS, topk) on this handle fits one warp's shared memory, and the plan it would run with:
// out = {ring depth, result heap in shared memory (1) or global memory (0), per-warp bytes, neighbour slots, row stride}.
// Handles of the reference library report that they fit (out all zeros): they search on the CPU.
int pb200_hnsw_search_fits(void* model_ptr, uint32_t efS, uint32_t topk, uint32_t* out) {
    PB200_API_BEGIN
    for (int i = 0; i < 5; ++i) out[i] = 0u;
    if (!hnsw_is_ours(model_ptr)) return 1;
    PB200_LOCK(hnsw_of(model_ptr))
    const pb200::HnswEngine& e = hnsw_of(model_ptr).primary();
    const pb200::HnswPlan p = e.search_plan(efS, topk);
    out[0] = static_cast<uint32_t>(p.stages); out[1] = p.heap_in_smem ? 1u : 0u; out[2] = p.per_warp; out[3] = p.nbmax;
    out[4] = e.sparse() ? 0u : pb200::dense_vstride(e.host().feat_dim);
    return p.fits ? 1 : 0;
    PB200_API_END("pb200_hnsw_search_fits")
}

// Host-only, no handle: the same plan for a dense index of width feat_dim whose longest neighbour list (level 0 or above) has
// max_degree entries, at ring depth setting `stages`; out as above.
int pb200_hnsw_dense_plan(uint32_t feat_dim, uint32_t max_degree, int stages, uint32_t efS, uint32_t topk, uint32_t* out) {
    const uint32_t vstride = pb200::dense_vstride(feat_dim);
    const pb200::HnswPlan p = pb200::hnsw_plan(false, vstride, max_degree, stages, std::max(efS, topk), 0u);
    out[0] = static_cast<uint32_t>(p.stages); out[1] = p.heap_in_smem ? 1u : 0u; out[2] = p.per_warp; out[3] = p.nbmax;
    out[4] = vstride;
    return p.fits ? 1 : 0;
}

void pb200_hnsw_get_counters(void* model_ptr, uint64_t* out) {
    PB200_API_BEGIN
    PB200_LOCK(hnsw_of(model_ptr))
    auto c = hnsw_of(model_ptr).primary().counters();
    out[0] = c.n_dist; out[1] = c.n_expand; out[2] = c.n_hops; out[3] = c.n_queries;
    PB200_API_END("pb200_hnsw_get_counters")
}

uint64_t pb200_hnsw_sparse_entries(void* model_ptr) {
    PB200_API_BEGIN
    PB200_LOCK(hnsw_of(model_ptr))
    return hnsw_of(model_ptr).primary().counters().n_entries;
    PB200_API_END("pb200_hnsw_sparse_entries")
}

uint32_t pb200_hnsw_vcap_retries(void* ptr) {
    PB200_API_BEGIN
    return hnsw_of(ptr).primary().vcap_retries();
    PB200_API_END("pb200_hnsw_vcap_retries")
}

uint32_t pb200_hnsw_replicas(void* ptr) {
    PB200_API_BEGIN
    return static_cast<uint32_t>(hnsw_of(ptr).engines.size());
    PB200_API_END("pb200_hnsw_replicas")
}

// host-only ingest of an HNSW index (no CUDA calls): validates config.json + index.mmap_store exactly like the loader does and
// reports what it found.  Returns 0, or 1 with the reason on stderr (wrong index type, version, truncated records ...).
int pb200_hnsw_host_info(const char* model_dir, int metric, int sparse, uint64_t* out) {
    try {
        auto ix = pb200::load_hnsw_index(model_dir, metric, false, sparse != 0);
        uint64_t entries = 0, degree_sum = 0;
        for (uint32_t i = 0; i < ix->num_node; ++i) {
            degree_sum += std::min(ix->l0_neighborhood(i)[0], ix->l0_max_degree);
            if (ix->sparse) {
                const float* v; const uint32_t* c;
                const uint32_t len = ix->l0_sparse_row(i, &v, &c);
                for (uint32_t j = 1; j < len; ++j)
                    if (c[j] <= c[j - 1]) throw std::runtime_error("hnsw index: a stored row does not have strictly ascending indices");
                if (len && c[len - 1] >= ix->feat_dim) throw std::runtime_error("hnsw index: a stored index is out of range");
                entries += len;
            } else {
                entries += ix->feat_dim;
            }
        }
        out[0] = ix->num_node; out[1] = ix->feat_dim; out[2] = ix->maxM; out[3] = ix->maxM0; out[4] = ix->max_level;
        out[5] = ix->init_node; out[6] = entries; out[7] = degree_sum;
        return 0;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "pb200_hnsw_host_info: %s\n", e.what());
        return 1;
    }
}

void pb200_hnsw_get_info(void* model_ptr, uint64_t* out) {
    PB200_API_BEGIN
    auto& e = hnsw_of(model_ptr).primary();
    const auto& h = e.host();
    out[0] = h.num_node; out[1] = h.feat_dim; out[2] = h.maxM; out[3] = h.maxM0; out[4] = h.max_level; out[5] = h.init_node;
    out[6] = e.index_bytes(); out[7] = e.launches();
    PB200_API_END("pb200_hnsw_get_info")
}

}  // extern "C"

// ------------------------------------------------ PairwiseANN ---------------------------------------------------
// Every handle and searcher token comes from this library: train (a deep copy, pairwise.hpp:245-263) is served here too.

namespace {

struct PairwiseHandle {
    std::unique_ptr<pb200::PairwiseModel> model;
};

struct PairwiseSearchers {  // the reference's vector<Searcher>: here one stream + scratch, calls serialised on the token
    std::unique_ptr<pb200::PairwiseSearcher> searcher;
    std::mutex mu;
};

pb200::PairwiseModel& pairwise_of(void* ptr) {
    if (!ptr) throw std::runtime_error("null PairwiseANN handle");
    return *static_cast<PairwiseHandle*>(ptr)->model;
}

PairwiseSearchers& pairwise_searchers_of(void* ptr) {
    if (!ptr) throw std::runtime_error("null PairwiseANN searchers token");
    return *static_cast<PairwiseSearchers*>(ptr);
}

void* pairwise_wrap(std::unique_ptr<pb200::PairwiseHostModel> host) {
    auto h = std::make_unique<PairwiseHandle>();
    h->model = std::make_unique<pb200::PairwiseModel>(std::move(host));
    return h.release();
}

void pairwise_check_type(void* model_ptr, bool sparse) {
    if (pairwise_of(model_ptr).host().sparse != sparse) throw std::runtime_error("PairwiseANN handle of the other data type");
}

}  // namespace

extern "C" {

#define PB200_PAIRWISE_API(SUFFIX, MAT_T, SPARSE)                                                                          \
    void* c_pairwise_ann_load##SUFFIX(const char* model_dir, const bool lazy_load) {                                      \
        PB200_API_BEGIN                                                                                                   \
        return pairwise_wrap(pb200::load_pairwise_model(model_dir, SPARSE, lazy_load));                                   \
        PB200_API_END("c_pairwise_ann_load" #SUFFIX)                                                                      \
    }                                                                                                                     \
    void c_pairwise_ann_save##SUFFIX(void* model_ptr, const char* model_dir) {                                            \
        PB200_API_BEGIN                                                                                                   \
        pairwise_check_type(model_ptr, SPARSE);                                                                           \
        pb200::save_pairwise_model(pairwise_of(model_ptr).host(), model_dir);                                             \
        PB200_API_END("c_pairwise_ann_save" #SUFFIX)                                                                      \
    }                                                                                                                     \
    void c_pairwise_ann_destruct##SUFFIX(void* model_ptr) {                                                               \
        PB200_API_BEGIN                                                                                                   \
        delete static_cast<PairwiseHandle*>(model_ptr);                                                                   \
        PB200_API_END("c_pairwise_ann_destruct" #SUFFIX)                                                                  \
    }                                                                                                                     \
    void* c_pairwise_ann_searchers_create##SUFFIX(void* model_ptr, uint32_t num_searcher) {                               \
        PB200_API_BEGIN                                                                                                   \
        (void)num_searcher; /* one token serves any number of pairs: the GPU kernels balance them */                      \
        pairwise_check_type(model_ptr, SPARSE);                                                                           \
        auto t = std::make_unique<PairwiseSearchers>();                                                                   \
        t->searcher = std::make_unique<pb200::PairwiseSearcher>(&pairwise_of(model_ptr), g_device.load());                \
        return t.release();                                                                                               \
        PB200_API_END("c_pairwise_ann_searchers_create" #SUFFIX)                                                          \
    }                                                                                                                     \
    void c_pairwise_ann_searchers_destruct##SUFFIX(void* searchers_ptr) {                                                 \
        PB200_API_BEGIN                                                                                                   \
        delete static_cast<PairwiseSearchers*>(searchers_ptr);                                                            \
        PB200_API_END("c_pairwise_ann_searchers_destruct" #SUFFIX)                                                        \
    }                                                                                                                     \
    void* c_pairwise_ann_train##SUFFIX(const MAT_T* pX, const ScipyCscF32* pY) {                                          \
        PB200_API_BEGIN                                                                                                   \
        return pairwise_wrap(                                                                                             \
            pb200::pairwise_train(host_matrix(pX), pY->rows, pY->cols, pY->col_ptr, pY->row_idx, pY->val));               \
        PB200_API_END("c_pairwise_ann_train" #SUFFIX)                                                                     \
    }                                                                                                                     \
    void c_pairwise_ann_predict##SUFFIX(void* searchers_ptr, uint32_t batch_size, uint32_t only_topk, const MAT_T* pQ,    \
                                        uint32_t* label_keys, uint32_t* ret_Imat, uint32_t* ret_Mmat, float* ret_Dmat,    \
                                        float* ret_Vmat, const bool is_same_input) {                                      \
        PB200_API_BEGIN                                                                                                   \
        auto& t = pairwise_searchers_of(searchers_ptr);                                                                   \
        std::lock_guard<std::mutex> lock(t.mu);                                                                           \
        t.searcher->predict(batch_size, only_topk, host_matrix(pQ), label_keys, ret_Imat, ret_Mmat, ret_Dmat, ret_Vmat,   \
                            is_same_input);                                                                               \
        PB200_API_END("c_pairwise_ann_predict" #SUFFIX)                                                                   \
    }

PB200_PAIRWISE_API(_drm_ip_f32, ScipyDrmF32, false)
PB200_PAIRWISE_API(_csr_ip_f32, ScipyCsrF32, true)

void pb200_pairwise_ann_get_counters(void* searchers_ptr, uint64_t* out) {
    PB200_API_BEGIN
    auto& t = pairwise_searchers_of(searchers_ptr);
    std::lock_guard<std::mutex> lock(t.mu);
    const auto c = t.searcher->counters();
    out[0] = c.pairs; out[1] = c.n_dist; out[2] = c.n_entries; out[3] = c.replays;
    PB200_API_END("pb200_pairwise_ann_get_counters")
}

double pb200_pairwise_ann_kernel_ms(void* searchers_ptr) {
    PB200_API_BEGIN
    auto& t = pairwise_searchers_of(searchers_ptr);
    std::lock_guard<std::mutex> lock(t.mu);
    return t.searcher->last_kernel_ms();
    PB200_API_END("pb200_pairwise_ann_kernel_ms")
}

void pb200_pairwise_ann_launch_info(void* searchers_ptr, uint64_t* out) {
    PB200_API_BEGIN
    auto& t = pairwise_searchers_of(searchers_ptr);
    std::lock_guard<std::mutex> lock(t.mu);
    t.searcher->launch_info(out);
    PB200_API_END("pb200_pairwise_ann_launch_info")
}

int pb200_pairwise_ann_dense_fits(uint32_t feat_dim, uint32_t* out) {
    const uint32_t vstride = pb200::dense_vstride(feat_dim);
    const pb200::PairwisePlan plan = pb200::pairwise_plan(false, vstride, 0);
    if (out) { out[0] = static_cast<uint32_t>(plan.stages); out[1] = plan.per_warp; out[2] = vstride; }
    return plan.fits ? 1 : 0;
}

int pb200_pairwise_ann_host_info(const char* model_dir, int sparse, uint64_t* out) {
    try {
        auto m = pb200::load_pairwise_model(model_dir, sparse != 0, false);
        uint64_t longest = 0;
        for (uint32_t l = 0; l < m->num_label_keys; ++l) longest = std::max<uint64_t>(longest, m->col_len(l));
        out[0] = m->num_input_keys; out[1] = m->num_label_keys; out[2] = m->feat_dim; out[3] = m->nnz_y; out[4] = m->nnz_x;
        out[5] = longest;
        return 0;
    } catch (const std::exception& e) {
        std::fprintf(stderr, "pb200_pairwise_ann_host_info: %s\n", e.what());
        return 1;
    }
}

// ------------------------------------------------ sparse x sparse products ------------------------------------------
// The calling thread's last product: pb200_spmm_last_info / pb200_spmm_last_kernel_ms.
static thread_local uint64_t t_spmm_info[pb200::kSpmmInfoLen] = {};
static thread_local double t_spmm_kernel_ms = 0.0;

// csr: Z = X Y row by row of X (rows of Y); csc: column by column of Y (columns of X) -- libpecos.cpp:320-335
static void sparse_matmul(const uint32_t x_rows, const uint32_t x_cols, const uint32_t y_rows, const uint32_t y_cols,
                          const pb200::SpmmOperand& a, const pb200::SpmmOperand& b, uint32_t width, bool col_major,
                          py_sparse_allocator_t pred_alloc, bool eliminate_zeros, bool sorted_indices) {
    if (x_cols != y_rows)
        throw std::runtime_error("X.cols = " + std::to_string(x_cols) + " != Y.rows = " + std::to_string(y_rows));
    pb200::spmm_run(g_device.load(), a, b, width, col_major, x_rows, y_cols, pred_alloc, eliminate_zeros, sorted_indices,
                    t_spmm_info, &t_spmm_kernel_ms);
}

void c_sparse_matmul_csr_f32(const ScipyCsrF32* pX, const ScipyCsrF32* pY, py_sparse_allocator_t pred_alloc,
                             const bool eliminate_zeros, const bool sorted_indices, int threads) {
    PB200_API_BEGIN
    (void)threads;
    sparse_matmul(pX->rows, pX->cols, pY->rows, pY->cols, {pX->rows, pX->row_ptr, pX->col_idx, pX->val},
                  {pY->rows, pY->row_ptr, pY->col_idx, pY->val}, pY->cols, false, pred_alloc, eliminate_zeros, sorted_indices);
    PB200_API_END("c_sparse_matmul_csr_f32")
}

void c_sparse_matmul_csc_f32(const ScipyCscF32* pX, const ScipyCscF32* pY, py_sparse_allocator_t pred_alloc,
                             const bool eliminate_zeros, const bool sorted_indices, int threads) {
    PB200_API_BEGIN
    (void)threads;
    sparse_matmul(pX->rows, pX->cols, pY->rows, pY->cols, {pY->cols, pY->col_ptr, pY->row_idx, pY->val},
                  {pX->cols, pX->col_ptr, pX->row_idx, pX->val}, pX->rows, true, pred_alloc, eliminate_zeros, sorted_indices);
    PB200_API_END("c_sparse_matmul_csc_f32")
}

int pb200_spmm_fits(uint32_t b_rows, uint64_t b_nnz, uint64_t* out) {
    const uint64_t need = (b_nnz >> 60) ? ~0ull : pb200::spmm_min_bytes(b_rows, b_nnz);
    size_t free_b = 0, total_b = 0;
    const bool ok = cudaSetDevice(g_device.load()) == cudaSuccess && cudaMemGetInfo(&free_b, &total_b) == cudaSuccess;
    if (!ok) cudaGetLastError();
    if (out) { out[0] = need; out[1] = ok ? free_b : 0; }
    return ok && need <= free_b ? 1 : 0;
}

void pb200_spmm_last_info(uint64_t* out) {
    for (int i = 0; i < pb200::kSpmmInfoLen; ++i) out[i] = t_spmm_info[i];
}

double pb200_spmm_last_kernel_ms(void) { return t_spmm_kernel_ms; }

}  // extern "C"
