// Sparse x sparse matrix product (see spmm_engine.h).  Two passes, because the caller allocates:
//   symbolic  per A row, the number of distinct output indices (the reference's col_ptr, matrix.hpp:1148-1190);
//   numeric   per A row, the exact fold, then the row's entries in ascending index order or in first-touch order.
// Every output entry has one owner (a lane, or a thread of a CTA) per step of the fold, and steps follow the reference's
// traversal order, so the sums are the reference's bit for bit.  B stays on the device for the whole call; A is streamed in
// row tiles that fit the workspace budget (PB200_SPMM_WORKSPACE_MB).
#include "spmm_engine.h"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "cuda_util.h"

namespace pb200 {
namespace {

constexpr uint32_t kEmpty = 0xFFFFFFFFu;  // no valid output index: widths are at most 2^32 - 1
constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int kWarpsPerCta = 4;           // warp tiers
constexpr int kCtaThreads = 256;          // CTA tiers
constexpr int kCtaWarps = kCtaThreads / 32;
constexpr uint32_t kCountSlots = 2 * kCountWarpMaxProducts;
constexpr uint32_t kFoldSlots = 2 * kFoldWarpMaxDistinct;
constexpr uint64_t kDefaultWorkspaceMB = 1024;
constexpr uint64_t kMinWorkspaceBytes = 64ull << 20;

__device__ __forceinline__ uint32_t slot_hash(uint32_t key, uint32_t log2) { return (key * 0x9E3779B1u) >> (32 - log2); }

// The reference's products and sums as x86 SSE computes them (mulss / addss, no FMA): the IEEE result, except for NaN
// results, where SSE returns the first NaN operand made quiet (the B value of a product, the new product of a sum: that
// is the operand order of the reference's compiled loop) or, when no operand is NaN (inf * 0, inf - inf), the default NaN
// 0xFFC00000.  The GPU would return 0x7FFFFFFF in every NaN case.
__device__ __forceinline__ float sse_nan(float first, float second) {
    if (isnan(first)) return __uint_as_float(__float_as_uint(first) | 0x00400000u);
    if (isnan(second)) return __uint_as_float(__float_as_uint(second) | 0x00400000u);
    return __uint_as_float(0xFFC00000u);
}
__device__ __forceinline__ float ref_mul(float a, float b) {
    const float r = __fmul_rn(a, b);
    return isnan(r) ? sse_nan(b, a) : r;
}
__device__ __forceinline__ float ref_add(float acc, float p) {
    const float r = __fadd_rn(acc, p);
    return isnan(r) ? sse_nan(p, acc) : r;
}

__device__ __forceinline__ unsigned lanemask_lt() { return (1u << (threadIdx.x & 31)) - 1u; }

// An open-addressing table (linear probing) of output index -> {value, first-touch rank}, in shared or global memory.
struct FoldTable {
    uint32_t* key;
    float* val;
    uint32_t* rank;
    uint32_t log2;  // slots = 1 << log2
};

__device__ __forceinline__ uint32_t find_or_insert(uint32_t* keys, uint32_t log2, uint32_t key, bool& inserted) {
    const uint32_t mask = (1u << log2) - 1u;
    uint32_t h = slot_hash(key, log2);
    while (true) {
        const uint32_t old = atomicCAS(&keys[h], kEmpty, key);
        if (old == kEmpty) { inserted = true; return h; }
        if (old == key) { inserted = false; return h; }
        h = (h + 1) & mask;
    }
}

__device__ __forceinline__ uint32_t find_slot(const uint32_t* keys, uint32_t log2, uint32_t key) {
    const uint32_t mask = (1u << log2) - 1u;
    uint32_t h = slot_hash(key, log2);
    while (keys[h] != key) h = (h + 1) & mask;
    return h;
}

__device__ __forceinline__ uint32_t table_log2(uint32_t distinct) {
    uint32_t log2 = 5;  // at least 32 slots, at least twice the distinct outputs
    while ((1ull << log2) < 2ull * distinct) ++log2;
    return log2;
}

// One warp applies a_s x (B row [q0, q1)) to t in stored order: lanes take consecutive entries, entries of one index in the
// same 32-entry step are applied in lane order (__match_any_sync), steps one after the other.  New indices get the next
// first-touch ranks in lane order.  mark: also set each new index's bit in `bitmap`.  Returns the rank counter after.
__device__ uint32_t warp_apply_row(const FoldTable& t, float a, const uint32_t* __restrict__ b_idx, const float* __restrict__ b_val,
                                   uint64_t q0, uint64_t q1, uint32_t rank, bool mark, uint32_t* bitmap) {
    const uint32_t lane = threadIdx.x & 31;
    for (uint64_t base = q0; base < q1; base += 32) {
        const uint64_t q = base + lane;
        const bool on = q < q1;
        const uint32_t key = on ? b_idx[q] : kEmpty;
        const float prod = on ? ref_mul(a, b_val[q]) : 0.0f;
        const unsigned grp = __match_any_sync(kFull, key);
        const int leader = __ffs(grp) - 1;
        bool inserted = false;
        uint32_t slot = 0;
        if (on && static_cast<int>(lane) == leader) slot = find_or_insert(t.key, t.log2, key, inserted);
        slot = __shfl_sync(kFull, slot, leader);
        const unsigned fresh = __ballot_sync(kFull, inserted);
        if (inserted) {
            t.rank[slot] = rank + __popc(fresh & lanemask_lt());
            if (mark) atomicOr(&bitmap[key >> 5], 1u << (key & 31));
        }
        rank += __popc(fresh);
        const uint32_t pos = __popc(grp & lanemask_lt());
        const uint32_t depth = __reduce_max_sync(kFull, on ? static_cast<uint32_t>(__popc(grp)) : 0u);
        for (uint32_t d = 0; d < depth; ++d) {
            if (on && pos == d) t.val[slot] = ref_add(t.val[slot], prod);
            __syncwarp();
        }
    }
    return rank;
}

// Exclusive prefix over the CTA of one u32 per thread; *total gets the sum.  Uses sh[kCtaWarps]; starts and ends with a barrier.
__device__ __forceinline__ uint32_t cta_exclusive(uint32_t v, uint32_t* sh, uint32_t* total) {
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const uint32_t n = __shfl_up_sync(kFull, inc, o);
        if (lane >= static_cast<uint32_t>(o)) inc += n;
    }
    __syncthreads();
    if (lane == 31) sh[warp] = inc;
    __syncthreads();
    uint32_t before = 0, sum = 0;
#pragma unroll
    for (int w = 0; w < kCtaWarps; ++w) {
        if (w < static_cast<int>(warp)) before += sh[w];
        sum += sh[w];
    }
    *total = sum;
    __syncthreads();
    return before + inc - v;
}

}  // namespace

// Kernels keep stable (non-anonymous) names for profiles.
// Per B row: 1 if its indices are strictly ascending (no repeats, so one step of a CTA may apply the row in parallel).
// Sets *bad when an index is not below the output width.
__global__ void __launch_bounds__(256) spmm_brow_flags_kernel(const uint64_t* __restrict__ b_ptr, const uint32_t* __restrict__ b_idx,
                                                              uint32_t b_rows, uint32_t width, uint8_t* __restrict__ canon,
                                                              uint32_t* bad) {
    const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= b_rows) return;
    bool ok = true, in_range = true;
    uint32_t prev = 0;
    for (uint64_t q = b_ptr[r]; q < b_ptr[r + 1]; ++q) {
        const uint32_t k = b_idx[q];
        if (k >= width) in_range = false;
        if (q > b_ptr[r] && k <= prev) ok = false;
        prev = k;
    }
    canon[r] = ok ? 1 : 0;
    if (!in_range) atomicOr(bad, 1u);
}

// Symbolic pass, short rows: one warp per row, a shared-memory hash set of kCountSlots indices.
__global__ void __launch_bounds__(kWarpsPerCta * 32) spmm_count_warp_kernel(
    const uint32_t* __restrict__ rows, uint32_t n, const uint64_t* __restrict__ a_ptr, uint64_t a_base,
    const uint32_t* __restrict__ a_idx, const uint64_t* __restrict__ b_ptr, const uint32_t* __restrict__ b_idx,
    uint32_t* __restrict__ distinct) {
    __shared__ uint32_t table[kWarpsPerCta][kCountSlots];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t k = blockIdx.x * kWarpsPerCta + warp;
    if (k >= n) return;
    const uint32_t r = rows[k];
    uint32_t* t = table[warp];
    for (uint32_t i = lane; i < kCountSlots; i += 32) t[i] = kEmpty;
    __syncwarp();
    constexpr uint32_t log2 = __builtin_ctz(kCountSlots);
    uint32_t count = 0;
    for (uint64_t s = a_ptr[r] - a_base; s < a_ptr[r + 1] - a_base; ++s) {
        const uint32_t b = a_idx[s];
        for (uint64_t q = b_ptr[b] + lane; q < b_ptr[b + 1]; q += 32) {
            bool inserted = false;
            find_or_insert(t, log2, b_idx[q], inserted);
            count += inserted;
        }
    }
    count = __reduce_add_sync(kFull, count);
    if (lane == 0) distinct[r] = count;
}

// Symbolic pass, long rows: one CTA per row (claimed from *next), a global bitmap of the output width per CTA.  Counting is
// order-free, so warps take A entries round-robin.  The bitmap is cleared again by walking the same entries.
__global__ void __launch_bounds__(kCtaThreads) spmm_count_cta_kernel(
    const uint32_t* __restrict__ rows, uint32_t n, const uint64_t* __restrict__ a_ptr, uint64_t a_base,
    const uint32_t* __restrict__ a_idx, const uint64_t* __restrict__ b_ptr, const uint32_t* __restrict__ b_idx,
    uint32_t* __restrict__ bitmaps, uint64_t words, uint32_t* next, uint32_t* __restrict__ distinct) {
    __shared__ uint32_t claim;
    __shared__ uint32_t sh[kCtaWarps];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t* bm = bitmaps + blockIdx.x * words;
    while (true) {
        if (threadIdx.x == 0) claim = atomicAdd(next, 1u);
        __syncthreads();
        const uint32_t k = claim;
        __syncthreads();
        if (k >= n) return;
        const uint32_t r = rows[k];
        const uint64_t s0 = a_ptr[r] - a_base, s1 = a_ptr[r + 1] - a_base;
        uint32_t count = 0;
        for (uint64_t s = s0 + warp; s < s1; s += kCtaWarps) {
            const uint32_t b = a_idx[s];
            for (uint64_t q = b_ptr[b] + lane; q < b_ptr[b + 1]; q += 32) {
                const uint32_t key = b_idx[q], bit = 1u << (key & 31);
                count += (atomicOr(&bm[key >> 5], bit) & bit) == 0;
            }
        }
        uint32_t total = 0;
        cta_exclusive(count, sh, &total);
        if (threadIdx.x == 0) distinct[r] = total;
        for (uint64_t s = s0 + warp; s < s1; s += kCtaWarps) {
            const uint32_t b = a_idx[s];
            for (uint64_t q = b_ptr[b] + lane; q < b_ptr[b + 1]; q += 32) bm[b_idx[q] >> 5] = 0;
        }
        __syncthreads();
    }
}

// Writes a folded warp-tier row: ascending indices (bitonic sort of {index, value bits} in `buf`) or first-touch order.
__device__ void warp_emit(const FoldTable& t, uint32_t d, unsigned long long* buf, bool sorted, uint32_t* __restrict__ out_idx,
                          float* __restrict__ out_val) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t slots = 1u << t.log2;
    if (!sorted) {
        for (uint32_t i = lane; i < slots; i += 32)
            if (t.key[i] != kEmpty) {
                out_idx[t.rank[i]] = t.key[i];
                out_val[t.rank[i]] = t.val[i];
            }
        return;
    }
    // buf aliases the rank array, which a sorted row does not read
    uint32_t n = 32;
    while (n < d) n <<= 1;
    uint32_t base = 0;
    for (uint32_t i = lane; i < slots; i += 32) {
        const bool full = t.key[i] != kEmpty;
        const unsigned b = __ballot_sync(kFull, full);
        if (full) buf[base + __popc(b & lanemask_lt())] = (static_cast<unsigned long long>(t.key[i]) << 32) | __float_as_uint(t.val[i]);
        base += __popc(b);
    }
    for (uint32_t i = d + lane; i < n; i += 32) buf[i] = ~0ull;
    __syncwarp();
    for (uint32_t k = 2; k <= n; k <<= 1)
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = lane; i < n; i += 32) {
                const uint32_t p = i ^ j;
                if (p > i) {
                    const unsigned long long x = buf[i], y = buf[p];
                    if ((x > y) == ((i & k) == 0)) { buf[i] = y; buf[p] = x; }
                }
            }
            __syncwarp();
        }
    for (uint32_t i = lane; i < d; i += 32) {
        out_idx[i] = static_cast<uint32_t>(buf[i] >> 32);
        out_val[i] = __uint_as_float(static_cast<uint32_t>(buf[i]));
    }
}

// Numeric pass, short rows: one warp per row, the accumulator in shared memory (kFoldSlots slots).
__global__ void __launch_bounds__(kWarpsPerCta * 32) spmm_fold_warp_kernel(
    const uint32_t* __restrict__ rows, uint32_t n, const uint64_t* __restrict__ a_ptr, uint64_t a_base,
    const uint32_t* __restrict__ a_idx, const float* __restrict__ a_val, const uint64_t* __restrict__ b_ptr,
    const uint32_t* __restrict__ b_idx, const float* __restrict__ b_val, const uint32_t* __restrict__ distinct,
    const uint64_t* __restrict__ out_off, uint64_t out_base, uint32_t* __restrict__ out_idx, float* __restrict__ out_val,
    int sorted) {
    __shared__ uint32_t skey[kWarpsPerCta][kFoldSlots];
    __shared__ float sval[kWarpsPerCta][kFoldSlots];
    __shared__ __align__(8) uint32_t srank[kWarpsPerCta][kFoldSlots];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t k = blockIdx.x * kWarpsPerCta + warp;
    if (k >= n) return;
    const uint32_t r = rows[k];
    const uint32_t d = distinct[r];
    const FoldTable t{skey[warp], sval[warp], srank[warp], table_log2(d)};
    for (uint32_t i = lane; i < (1u << t.log2); i += 32) { t.key[i] = kEmpty; t.val[i] = 0.0f; }
    __syncwarp();
    uint32_t rank = 0;
    for (uint64_t s = a_ptr[r] - a_base; s < a_ptr[r + 1] - a_base; ++s) {
        const uint32_t b = a_idx[s];
        rank = warp_apply_row(t, a_val[s], b_idx, b_val, b_ptr[b], b_ptr[b + 1], rank, false, nullptr);
    }
    __syncwarp();
    const uint64_t o = out_off[r] - out_base;
    warp_emit(t, d, reinterpret_cast<unsigned long long*>(srank[warp]), sorted != 0, out_idx + o, out_val + o);
}

// Numeric pass, long rows: one CTA per row (claimed from *next), the accumulator in global memory at tab_off[k] (2-4x the
// row's distinct outputs).  A strictly ascending B row is applied by all threads in 256-entry steps; any other B row by warp 0
// alone, as in the warp tier.  Sorted rows set a bit per index in the CTA's bitmap and are written out by scanning it.
__global__ void __launch_bounds__(kCtaThreads) spmm_fold_cta_kernel(
    const uint32_t* __restrict__ rows, uint32_t n, const uint64_t* __restrict__ a_ptr, uint64_t a_base,
    const uint32_t* __restrict__ a_idx, const float* __restrict__ a_val, const uint64_t* __restrict__ b_ptr,
    const uint32_t* __restrict__ b_idx, const float* __restrict__ b_val, const uint8_t* __restrict__ canon,
    const uint32_t* __restrict__ distinct, const uint64_t* __restrict__ out_off, uint64_t out_base,
    uint32_t* __restrict__ out_idx, float* __restrict__ out_val, const uint64_t* __restrict__ tab_off, uint32_t* tkey,
    float* tval, uint32_t* trank, uint32_t* bitmaps, uint64_t words, uint32_t* next, int sorted) {
    __shared__ uint32_t claim, rank_sh;
    __shared__ uint32_t sh[kCtaWarps];
    const uint32_t warp = threadIdx.x >> 5;
    uint32_t* bm = bitmaps + blockIdx.x * words;
    while (true) {
        if (threadIdx.x == 0) { claim = atomicAdd(next, 1u); rank_sh = 0; }
        __syncthreads();
        const uint32_t k = claim;
        if (k >= n) return;
        const uint32_t r = rows[k];
        const uint32_t d = distinct[r];
        const FoldTable t{tkey + tab_off[k], tval + tab_off[k], trank + tab_off[k], table_log2(d)};
        const uint32_t slots = 1u << t.log2;
        for (uint32_t i = threadIdx.x; i < slots; i += kCtaThreads) { t.key[i] = kEmpty; t.val[i] = 0.0f; }
        __syncthreads();
        for (uint64_t s = a_ptr[r] - a_base; s < a_ptr[r + 1] - a_base; ++s) {
            const uint32_t b = a_idx[s];
            const float a = a_val[s];
            const uint64_t q0 = b_ptr[b], q1 = b_ptr[b + 1];
            if (canon[b]) {
                for (uint64_t base = q0; base < q1; base += kCtaThreads) {
                    const uint64_t q = base + threadIdx.x;
                    bool inserted = false;
                    uint32_t key = 0, slot = 0;
                    float prod = 0.0f;
                    if (q < q1) {
                        key = b_idx[q];
                        prod = ref_mul(a, b_val[q]);
                        slot = find_or_insert(t.key, t.log2, key, inserted);
                    }
                    uint32_t total = 0;
                    const uint32_t before = cta_exclusive(inserted ? 1u : 0u, sh, &total);
                    if (inserted) {
                        t.rank[slot] = rank_sh + before;
                        if (sorted) atomicOr(&bm[key >> 5], 1u << (key & 31));
                    }
                    if (q < q1) t.val[slot] = ref_add(t.val[slot], prod);
                    __syncthreads();
                    if (threadIdx.x == 0) rank_sh += total;
                    __syncthreads();
                }
            } else {
                if (warp == 0) {
                    const uint32_t rk = warp_apply_row(t, a, b_idx, b_val, q0, q1, rank_sh, sorted != 0, bm);
                    __syncwarp();
                    if (threadIdx.x == 0) rank_sh = rk;
                }
                __syncthreads();
            }
        }
        const uint64_t o = out_off[r] - out_base;
        if (!sorted) {
            for (uint32_t i = threadIdx.x; i < slots; i += kCtaThreads)
                if (t.key[i] != kEmpty) {
                    out_idx[o + t.rank[i]] = t.key[i];
                    out_val[o + t.rank[i]] = t.val[i];
                }
        } else {
            uint32_t written = 0;
            for (uint64_t w0 = 0; w0 < words; w0 += kCtaThreads) {
                const uint64_t w = w0 + threadIdx.x;
                uint32_t bits = w < words ? bm[w] : 0u;
                uint32_t total = 0;
                uint32_t pos = written + cta_exclusive(__popc(bits), sh, &total);
                if (bits) bm[w] = 0;
                while (bits) {
                    const uint32_t key = static_cast<uint32_t>(w) * 32 + (__ffs(bits) - 1);
                    bits &= bits - 1;
                    const uint32_t slot = find_slot(t.key, t.log2, key);
                    out_idx[o + pos] = key;
                    out_val[o + pos] = t.val[slot];
                    ++pos;
                }
                written += total;
            }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------------------ host side
namespace {


// Per-device state: B, the current A tile, the workspace and the staging buffers.  One call at a time per device.
struct SpmmDevice {
    std::mutex mu;
    bool ready = false;
    int sms = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    DeviceBuffer<uint64_t> a_ptr, b_ptr, out_off, tab_off;
    DeviceBuffer<uint32_t> a_idx, b_idx, rows, distinct, tkey, trank, bitmaps, out_idx, counters;
    DeviceBuffer<float> a_val, b_val, tval, out_val;
    DeviceBuffer<uint8_t> canon;
    PinnedBuffer<uint32_t> h_idx;
    PinnedBuffer<float> h_val;
};

SpmmDevice& spmm_device(int device) {
    static std::mutex mu;
    static std::vector<std::unique_ptr<SpmmDevice>> devs;
    std::lock_guard<std::mutex> lock(mu);
    if (device < 0) throw std::runtime_error("bad device id");
    if (devs.size() <= static_cast<size_t>(device)) devs.resize(device + 1);
    if (!devs[device]) devs[device] = std::make_unique<SpmmDevice>();
    return *devs[device];
}

uint64_t workspace_budget() {
    const char* env = std::getenv("PB200_SPMM_WORKSPACE_MB");
    uint64_t mb = kDefaultWorkspaceMB;
    if (env && *env) {
        char* end = nullptr;
        const unsigned long long v = std::strtoull(env, &end, 10);
        if (*end != 0 || v == 0) throw std::runtime_error(std::string("PB200_SPMM_WORKSPACE_MB: bad value '") + env + "'");
        mb = v;
    }
    return mb << 20;
}

uint32_t table_slots(uint32_t distinct) {
    uint64_t slots = 32;
    while (slots < 2ull * distinct) slots <<= 1;
    return static_cast<uint32_t>(slots);
}

// consecutive rows [begin, end) whose cost(i) sums to at most budget; a row costlier than the budget is a tile of its own
template <typename Cost>
std::vector<std::pair<uint32_t, uint32_t>> make_tiles(uint32_t rows, uint64_t budget, Cost&& cost) {
    std::vector<std::pair<uint32_t, uint32_t>> tiles;
    uint32_t begin = 0;
    uint64_t sum = 0;
    for (uint32_t i = 0; i < rows; ++i) {
        const uint64_t c = cost(i);
        if (i > begin && sum + c > budget) { tiles.emplace_back(begin, i); begin = i; sum = 0; }
        sum += c;
    }
    if (rows > begin) tiles.emplace_back(begin, rows);
    return tiles;
}

uint32_t blocks_for(uint64_t n, uint64_t per) { return static_cast<uint32_t>((n + per - 1) / per); }

}  // namespace

uint64_t spmm_min_bytes(uint32_t b_rows, uint64_t b_nnz) {
    return 8ull * (static_cast<uint64_t>(b_rows) + 1) + 8ull * b_nnz + b_rows + kMinWorkspaceBytes;
}

void spmm_run(int device, const SpmmOperand& A, const SpmmOperand& B, uint32_t width, bool col_major, uint64_t alloc_rows,
              uint64_t alloc_cols, py_sparse_allocator_t pred_alloc, bool eliminate_zeros, bool sorted_indices,
              uint64_t* info, double* kernel_ms) {
    std::fill(info, info + kSpmmInfoLen, 0ull);
    *kernel_ms = 0.0;
    // ---- validation and products, on the host, before any launch
    if (A.rows && (!A.ptr || (A.ptr[A.rows] && (!A.idx || !A.val)))) throw std::runtime_error("null A arrays");
    if (!B.ptr) throw std::runtime_error("null B pointer array");
    if (B.ptr[B.rows] && (!B.idx || !B.val)) throw std::runtime_error("null B arrays");
    for (uint32_t k = 0; k < B.rows; ++k)
        if (B.ptr[k] > B.ptr[k + 1]) throw std::runtime_error("B pointers decrease at row " + std::to_string(k));
    std::vector<uint64_t> products(A.rows);
    uint64_t total_products = 0;
    for (uint32_t i = 0; i < A.rows; ++i) {
        if (A.ptr[i] > A.ptr[i + 1]) throw std::runtime_error("A pointers decrease at row " + std::to_string(i));
        uint64_t p = 0;
        for (uint64_t s = A.ptr[i]; s < A.ptr[i + 1]; ++s) {
            const uint32_t b = A.idx[s];
            if (b >= B.rows)
                throw std::runtime_error("index " + std::to_string(b) + " of the left operand is beyond the right operand's " +
                                         std::to_string(B.rows) + " rows");
            p += B.ptr[b + 1] - B.ptr[b];
        }
        products[i] = p;
        total_products += p;
    }
    const uint64_t budget = workspace_budget();
    info[0] = A.rows;
    info[1] = total_products;

    SpmmDevice& dev = spmm_device(device);
    std::lock_guard<std::mutex> lock(dev.mu);
    PB200_CUDA(cudaSetDevice(device));
    if (!dev.ready) {
        PB200_CUDA(cudaDeviceGetAttribute(&dev.sms, cudaDevAttrMultiProcessorCount, device));
        PB200_CUDA(cudaStreamCreateWithFlags(&dev.stream, cudaStreamNonBlocking));
        PB200_CUDA(cudaEventCreate(&dev.ev0));
        PB200_CUDA(cudaEventCreate(&dev.ev1));
        dev.ready = true;
    }
    cudaStream_t st = dev.stream;
    uint64_t launches = 0, tiles_run = 0;
    float ms_total = 0.0f;
    auto timed = [&](auto&& work) {
        PB200_CUDA(cudaEventRecord(dev.ev0, st));
        work();
        PB200_CUDA(cudaEventRecord(dev.ev1, st));
        PB200_CUDA(cudaEventSynchronize(dev.ev1));
        float ms = 0.0f;
        PB200_CUDA(cudaEventElapsedTime(&ms, dev.ev0, dev.ev1));
        ms_total += ms;
    };

    std::vector<uint32_t> distinct(A.rows, 0);
    const uint64_t words = (static_cast<uint64_t>(width) + 31) / 32;
    if (total_products > 0) {
        // ---- B, its row flags and the A pointers stay on the device for the whole call
        const uint64_t b_nnz = B.ptr[B.rows];
        dev.b_ptr.upload(B.ptr, B.rows + 1ull, st);
        dev.b_idx.upload(B.idx, b_nnz, st);
        dev.b_val.upload(B.val, b_nnz, st);
        dev.a_ptr.upload(A.ptr, A.rows + 1ull, st);
        dev.canon.reserve(B.rows);
        dev.counters.reserve(2);  // [0] CTA row claims, [1] out-of-range flag
        PB200_CUDA(cudaMemsetAsync(dev.counters.get(), 0, 2 * sizeof(uint32_t), st));
        if (B.rows) {
            spmm_brow_flags_kernel<<<blocks_for(B.rows, 256), 256, 0, st>>>(dev.b_ptr.get(), dev.b_idx.get(), B.rows, width,
                                                                           dev.canon.get(), dev.counters.get() + 1);
            PB200_CUDA(cudaGetLastError());
            ++launches;
        }
        uint32_t bad = 0;
        PB200_CUDA(cudaMemcpyAsync(&bad, dev.counters.get() + 1, sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        PB200_CUDA(cudaStreamSynchronize(st));
        if (bad) throw std::runtime_error("an index of the right operand is not below the output width " + std::to_string(width));
        dev.distinct.reserve(A.rows);
        PB200_CUDA(cudaMemsetAsync(dev.distinct.get(), 0, A.rows * sizeof(uint32_t), st));
        // CTA-tier workers: one output-width bitmap each, at most a quarter of the budget, at most 2 per SM
        const uint64_t bm_bytes = std::max<uint64_t>(words * 4, 4);
        const uint32_t slots_cta = static_cast<uint32_t>(
            std::max<uint64_t>(1, std::min<uint64_t>(2ull * dev.sms, (budget / 4) / bm_bytes)));
        dev.bitmaps.reserve(slots_cta * std::max<uint64_t>(words, 1));
        PB200_CUDA(cudaMemsetAsync(dev.bitmaps.get(), 0, slots_cta * bm_bytes, st));

        // ---- symbolic pass
        const uint64_t a_rows_cost = 8 + 4 + 4;
        const auto sym_tiles = make_tiles(A.rows, budget / 2, [&](uint32_t i) {
            return a_rows_cost + 4 * (A.ptr[i + 1] - A.ptr[i]);
        });
        std::vector<uint32_t> warp_rows, cta_rows;
        for (const auto& tile : sym_tiles) {
            warp_rows.clear();
            cta_rows.clear();
            for (uint32_t i = tile.first; i < tile.second; ++i) {
                if (products[i] == 0) continue;
                (products[i] <= kCountWarpMaxProducts ? warp_rows : cta_rows).push_back(i);
            }
            if (warp_rows.empty() && cta_rows.empty()) continue;
            const uint64_t a_base = A.ptr[tile.first], a_n = A.ptr[tile.second] - a_base;
            dev.a_idx.upload(A.idx + a_base, a_n, st);
            std::vector<uint32_t> lists(warp_rows);
            lists.insert(lists.end(), cta_rows.begin(), cta_rows.end());
            dev.rows.upload(lists.data(), lists.size(), st);
            PB200_CUDA(cudaMemsetAsync(dev.counters.get(), 0, sizeof(uint32_t), st));
            timed([&] {
                if (!warp_rows.empty()) {
                    spmm_count_warp_kernel<<<blocks_for(warp_rows.size(), kWarpsPerCta), kWarpsPerCta * 32, 0, st>>>(
                        dev.rows.get(), static_cast<uint32_t>(warp_rows.size()), dev.a_ptr.get(), a_base, dev.a_idx.get(),
                        dev.b_ptr.get(), dev.b_idx.get(), dev.distinct.get());
                    PB200_CUDA(cudaGetLastError());
                    ++launches;
                }
                if (!cta_rows.empty()) {
                    const uint32_t grid = std::min<uint64_t>(slots_cta, cta_rows.size());
                    spmm_count_cta_kernel<<<grid, kCtaThreads, 0, st>>>(
                        dev.rows.get() + warp_rows.size(), static_cast<uint32_t>(cta_rows.size()), dev.a_ptr.get(), a_base,
                        dev.a_idx.get(), dev.b_ptr.get(), dev.b_idx.get(), dev.bitmaps.get(), words, dev.counters.get(),
                        dev.distinct.get());
                    PB200_CUDA(cudaGetLastError());
                    ++launches;
                }
            });
            info[4] += warp_rows.size();
            info[5] += cta_rows.size();
            ++tiles_run;
        }
        PB200_CUDA(cudaMemcpyAsync(distinct.data(), dev.distinct.get(), A.rows * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        PB200_CUDA(cudaStreamSynchronize(st));
    }

    // ---- the caller allocates
    std::vector<uint64_t> off(A.rows + 1ull, 0);
    for (uint32_t i = 0; i < A.rows; ++i) off[i + 1] = off[i] + distinct[i];
    const uint64_t nnz = off[A.rows];
    uint64_t indices_addr = 0, indptr_addr = 0, data_addr = 0;
    pred_alloc(col_major, alloc_rows, alloc_cols, nnz, &indices_addr, &indptr_addr, &data_addr);
    uint32_t* z_idx = reinterpret_cast<uint32_t*>(indices_addr);
    uint64_t* z_ptr = reinterpret_cast<uint64_t*>(indptr_addr);
    float* z_val = reinterpret_cast<float*>(data_addr);
    info[2] = nnz;
    z_ptr[0] = 0;
    if (nnz == 0) {
        for (uint32_t i = 0; i < A.rows; ++i) z_ptr[i + 1] = 0;
        info[8] = tiles_run;
        info[9] = launches;
        *kernel_ms = ms_total;
        return;
    }

    // ---- numeric pass
    const auto cta_tier = [&](uint32_t i) {
        return distinct[i] > kFoldWarpMaxDistinct || products[i] > kFoldWarpMaxProducts;
    };
    const auto tiles = make_tiles(A.rows, budget, [&](uint32_t i) {
        return 8 + 8 * (A.ptr[i + 1] - A.ptr[i]) + 8ull * distinct[i] + (cta_tier(i) ? 12ull * table_slots(distinct[i]) : 0);
    });
    dev.out_off.upload(off.data(), A.rows + 1ull, st);
    const uint32_t slots_cta = static_cast<uint32_t>(
        std::max<uint64_t>(1, std::min<uint64_t>(2ull * dev.sms, (budget / 4) / std::max<uint64_t>(words * 4, 4))));
    uint64_t kept = 0;
    std::vector<uint32_t> warp_rows, cta_rows;
    std::vector<uint64_t> tab_off;
    for (const auto& tile : tiles) {
        warp_rows.clear();
        cta_rows.clear();
        tab_off.clear();
        uint64_t tab_n = 0;
        for (uint32_t i = tile.first; i < tile.second; ++i) {
            if (distinct[i] == 0) continue;
            if (cta_tier(i)) {
                cta_rows.push_back(i);
                tab_off.push_back(tab_n);
                tab_n += table_slots(distinct[i]);
            } else {
                warp_rows.push_back(i);
            }
        }
        const uint64_t o0 = off[tile.first], o_n = off[tile.second] - o0;
        if (o_n == 0) {
            for (uint32_t i = tile.first; i < tile.second; ++i) z_ptr[i + 1] = kept;
            continue;
        }
        const uint64_t a_base = A.ptr[tile.first], a_n = A.ptr[tile.second] - a_base;
        dev.a_idx.upload(A.idx + a_base, a_n, st);
        dev.a_val.upload(A.val + a_base, a_n, st);
        std::vector<uint32_t> lists(warp_rows);
        lists.insert(lists.end(), cta_rows.begin(), cta_rows.end());
        dev.rows.upload(lists.data(), lists.size(), st);
        dev.out_idx.reserve(o_n);
        dev.out_val.reserve(o_n);
        if (!cta_rows.empty()) {
            dev.tab_off.upload(tab_off.data(), tab_off.size(), st);
            dev.tkey.reserve(tab_n);
            dev.tval.reserve(tab_n);
            dev.trank.reserve(tab_n);
        }
        PB200_CUDA(cudaMemsetAsync(dev.counters.get(), 0, sizeof(uint32_t), st));
        timed([&] {
            if (!warp_rows.empty()) {
                spmm_fold_warp_kernel<<<blocks_for(warp_rows.size(), kWarpsPerCta), kWarpsPerCta * 32, 0, st>>>(
                    dev.rows.get(), static_cast<uint32_t>(warp_rows.size()), dev.a_ptr.get(), a_base, dev.a_idx.get(),
                    dev.a_val.get(), dev.b_ptr.get(), dev.b_idx.get(), dev.b_val.get(), dev.distinct.get(), dev.out_off.get(), o0,
                    dev.out_idx.get(), dev.out_val.get(), sorted_indices ? 1 : 0);
                PB200_CUDA(cudaGetLastError());
                ++launches;
            }
            if (!cta_rows.empty()) {
                const uint32_t grid = std::min<uint64_t>(slots_cta, cta_rows.size());
                spmm_fold_cta_kernel<<<grid, kCtaThreads, 0, st>>>(
                    dev.rows.get() + warp_rows.size(), static_cast<uint32_t>(cta_rows.size()), dev.a_ptr.get(), a_base,
                    dev.a_idx.get(), dev.a_val.get(), dev.b_ptr.get(), dev.b_idx.get(), dev.b_val.get(), dev.canon.get(),
                    dev.distinct.get(), dev.out_off.get(), o0, dev.out_idx.get(), dev.out_val.get(), dev.tab_off.get(),
                    dev.tkey.get(), dev.tval.get(), dev.trank.get(), dev.bitmaps.get(), words, dev.counters.get(),
                    sorted_indices ? 1 : 0);
                PB200_CUDA(cudaGetLastError());
                ++launches;
            }
        });
        info[6] += warp_rows.size();
        info[7] += cta_rows.size();
        ++tiles_run;
        // ---- through pinned staging into the caller's arrays (compacted when asked)
        dev.h_idx.reserve(o_n);
        dev.h_val.reserve(o_n);
        PB200_CUDA(cudaMemcpyAsync(dev.h_idx.get(), dev.out_idx.get(), o_n * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
        PB200_CUDA(cudaMemcpyAsync(dev.h_val.get(), dev.out_val.get(), o_n * sizeof(float), cudaMemcpyDeviceToHost, st));
        PB200_CUDA(cudaStreamSynchronize(st));
        const uint32_t* hi = dev.h_idx.get();
        const float* hv = dev.h_val.get();
        if (!eliminate_zeros) {
            std::memcpy(z_idx + o0, hi, o_n * sizeof(uint32_t));
            std::memcpy(z_val + o0, hv, o_n * sizeof(float));
            for (uint32_t i = tile.first; i < tile.second; ++i) z_ptr[i + 1] = off[i + 1];
            kept = off[tile.second];
        } else {
            for (uint32_t i = tile.first; i < tile.second; ++i) {
                for (uint64_t e = off[i] - o0; e < off[i + 1] - o0; ++e)
                    if (hv[e] != 0.0f) {  // +-0 go, NaN stays (the reference's `val != 0`)
                        z_idx[kept] = hi[e];
                        z_val[kept] = hv[e];
                        ++kept;
                    }
                z_ptr[i + 1] = kept;
            }
        }
    }
    info[3] = kept;
    info[8] = tiles_run;
    info[9] = launches;
    *kernel_ms = ms_total;
}

}  // namespace pb200
