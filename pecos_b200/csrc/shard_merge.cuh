// Exchange records and merge kernel of index sharding, shared by the XR-Linear engine (leaf layer split over GPUs) and the
// HNSW engine (one graph per shard).
//
// Every rank packs its local top-k into 16-byte {key, id, value} records, ONE all-gather concatenates them as
// [world][rows][stride], and shard_merge_packed_kernel selects the k largest keys per query.  Keys are globally unique (each
// engine embeds the candidate's global position or (rank, slot) in the low word) and key 0 marks an empty slot (a valid key's
// low word is never 0), so the merge is an exact arg-max selection and no per-query count array travels.
#pragma once

#include <cstdint>

namespace pb200 {

namespace {

constexpr int kSelWarps = 4;    // queries per CTA of the warp-per-query selection kernels
constexpr int kSelKeys = 1024;  // merge kernel capacity: world * stride keys per query (static shared memory)

struct __align__(16) ShardRecord {
    unsigned long long key;
    uint32_t id;
    float val;
};
static_assert(sizeof(ShardRecord) == 16, "shard record must stay 16 bytes");

// monotone float -> u32 map: a < b (as floats, -0.0 < +0.0) <=> orderable(a) < orderable(b)
__device__ __forceinline__ uint32_t orderable(float v) {
    const uint32_t u = __float_as_uint(v);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// Merge of the per-GPU top-k records gathered by ONE all-gather ([world][rows][stride]) into the global top-k: for each
// output rank, the lane holding the warp's largest key finds its slot and emits that record.  Writes out_cnt[q] and the
// first out_cnt[q] entries of row q (row stride k); the rest of the row is left as it was.
__global__ void __launch_bounds__(kSelWarps * 32)
shard_merge_packed_kernel(const ShardRecord* __restrict__ g_rec, const uint32_t world, const uint32_t rows, const uint32_t stride,
                          const uint32_t k, uint32_t* __restrict__ out_id, float* __restrict__ out_val, uint32_t* __restrict__ out_cnt) {
    constexpr unsigned kAll = 0xFFFFFFFFu;
    __shared__ unsigned long long s_keys[kSelWarps][kSelKeys];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const uint32_t q = blockIdx.x * kSelWarps + warp;
    if (q >= rows) return;
    unsigned long long* keys = s_keys[warp];
    const uint32_t n = world * stride;
    unsigned long long best = 0ull;
    uint32_t total = 0;
    for (uint32_t i = lane; i < n; i += 32) {
        const uint32_t g = i / stride, r = i - g * stride;
        const unsigned long long key = g_rec[(static_cast<uint64_t>(g) * rows + q) * stride + r].key;
        if (key) ++total;
        keys[i] = key;
        best = key > best ? key : best;
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) total += __shfl_xor_sync(kAll, total, d);
    __syncwarp();
    const uint32_t kk = min(k, total);
    if (lane == 0) out_cnt[q] = kk;
    for (uint32_t rnk = 0; rnk < kk; ++rnk) {
        unsigned long long top = best;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            const unsigned long long o = __shfl_xor_sync(kAll, top, d);
            top = o > top ? o : top;
        }
        uint32_t slot = 0xFFFFFFFFu;
        if (best == top) {
            for (uint32_t i = lane; i < n; i += 32) if (keys[i] == top) { slot = i; break; }
        }
        if (slot != 0xFFFFFFFFu) {
            const uint32_t g = slot / stride, r = slot - g * stride;
            const ShardRecord rc = g_rec[(static_cast<uint64_t>(g) * rows + q) * stride + r];
            out_id[static_cast<uint64_t>(q) * k + rnk] = rc.id;
            out_val[static_cast<uint64_t>(q) * k + rnk] = rc.val;
            keys[slot] = 0ull;
            best = 0ull;
            for (uint32_t i = lane; i < n; i += 32) { const unsigned long long key = keys[i]; best = key > best ? key : best; }
        }
        __syncwarp();
    }
}

}  // namespace

}  // namespace pb200
