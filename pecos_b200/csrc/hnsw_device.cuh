// Warp-level device helpers shared by the HNSW search kernels and the PairwiseANN kernels: the reference-order dense
// distance of a half-warp (with the bulk-copy row ring), the ordered sparse intersection, and the libstdc++ heap algorithms.
// See hnsw_engine.cu for how the search uses them.
#pragma once

#include "hnsw_engine.h"
#include "sparse_distance.cuh"

namespace pb200 {

namespace {

constexpr unsigned kFull = 0xFFFFFFFFu;

__device__ __forceinline__ float4 ld_stream_f4(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}

template <int METRIC>
__device__ __forceinline__ float chain_step(float acc, float x, float y) {
    if (METRIC == HNSW_IP) return __fadd_rn(acc, __fmul_rn(x, y));
    const float d = __fsub_rn(x, y);
    return __fadd_rn(acc, __fmul_rn(d, d));
}

// Distance between the staged (permuted) query and base vector `node`, computed by one half-warp.
// Every lane of the warp must call it; the result is valid on lanes 0 and 16 (hl == 0).
template <int METRIC, bool SMEM>
__device__ __forceinline__ float half_warp_distance(const HnswDev& ix, const float* qs, const float* row, int hl) {
    const float4* v4 = reinterpret_cast<const float4*>(row);
    const float4* q4 = reinterpret_cast<const float4*>(qs);
    const uint32_t nK = ix.main_pad >> 6;
    float acc = 0.0f;
    uint32_t K = 0;
    for (; K + 4 <= nK; K += 4) {
        const float4 y0 = SMEM ? v4[(K + 0) * 16 + hl] : ld_stream_f4(v4 + (K + 0) * 16 + hl);
        const float4 y1 = SMEM ? v4[(K + 1) * 16 + hl] : ld_stream_f4(v4 + (K + 1) * 16 + hl);
        const float4 y2 = SMEM ? v4[(K + 2) * 16 + hl] : ld_stream_f4(v4 + (K + 2) * 16 + hl);
        const float4 y3 = SMEM ? v4[(K + 3) * 16 + hl] : ld_stream_f4(v4 + (K + 3) * 16 + hl);
        const float4 x0 = q4[(K + 0) * 16 + hl], x1 = q4[(K + 1) * 16 + hl], x2 = q4[(K + 2) * 16 + hl], x3 = q4[(K + 3) * 16 + hl];
        acc = chain_step<METRIC>(acc, x0.x, y0.x); acc = chain_step<METRIC>(acc, x0.y, y0.y);
        acc = chain_step<METRIC>(acc, x0.z, y0.z); acc = chain_step<METRIC>(acc, x0.w, y0.w);
        acc = chain_step<METRIC>(acc, x1.x, y1.x); acc = chain_step<METRIC>(acc, x1.y, y1.y);
        acc = chain_step<METRIC>(acc, x1.z, y1.z); acc = chain_step<METRIC>(acc, x1.w, y1.w);
        acc = chain_step<METRIC>(acc, x2.x, y2.x); acc = chain_step<METRIC>(acc, x2.y, y2.y);
        acc = chain_step<METRIC>(acc, x2.z, y2.z); acc = chain_step<METRIC>(acc, x2.w, y2.w);
        acc = chain_step<METRIC>(acc, x3.x, y3.x); acc = chain_step<METRIC>(acc, x3.y, y3.y);
        acc = chain_step<METRIC>(acc, x3.z, y3.z); acc = chain_step<METRIC>(acc, x3.w, y3.w);
    }
    for (; K < nK; ++K) {
        const float4 y = SMEM ? v4[K * 16 + hl] : ld_stream_f4(v4 + K * 16 + hl);
        const float4 x = q4[K * 16 + hl];
        acc = chain_step<METRIC>(acc, x.x, y.x); acc = chain_step<METRIC>(acc, x.y, y.y);
        acc = chain_step<METRIC>(acc, x.z, y.z); acc = chain_step<METRIC>(acc, x.w, y.w);
    }
    // fold 16 partial sums -> 4:  (a[j] + a[4+j]) + (a[8+j] + a[12+j])   (x86.hpp:138-141)
    const float u = __fadd_rn(acc, __shfl_down_sync(kFull, acc, 4, 16));
    float s = __fadd_rn(u, __shfl_down_sync(kFull, u, 8, 16));
    const uint32_t tl = ix.tail_len;
    const float* yt = row + ix.main_pad;
    const float* xt = qs + ix.main_pad;
    const uint32_t g4 = tl >> 2;
    for (uint32_t g = 0; g < g4; ++g) {  // 4-wide remainder loop (x86.hpp:143-147), lanes 0..3 of the half-warp
        if (hl < 4) s = chain_step<METRIC>(s, xt[g * 4 + hl], yt[g * 4 + hl]);
    }
    const float s1 = __shfl_down_sync(kFull, s, 1, 16);
    const float s2 = __shfl_down_sync(kFull, s, 2, 16);
    const float s3 = __shfl_down_sync(kFull, s, 3, 16);
    float sum = __fadd_rn(__fadd_rn(__fadd_rn(s, s1), s2), s3);  // tmp_sum[0] + tmp_sum[1] + tmp_sum[2] + tmp_sum[3]
    for (uint32_t i = g4 * 4; i < tl; ++i) {  // scalar tail: fused multiply-add in the avx512f clone
        if (METRIC == HNSW_IP) sum = __fmaf_rn(xt[i], yt[i], sum);
        else { const float d = __fsub_rn(xt[i], yt[i]); sum = __fmaf_rn(d, d, sum); }
    }
    if (METRIC == HNSW_IP) return static_cast<float>(1.0 - static_cast<double>(sum));  // feat_vectors.hpp:138-141
    return sum;
}

// ---- bulk asynchronous copies (TMA engine, non-tensor form: SASS UBLKCP) + mbarrier completion -----------------------
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint32_t mbar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// one elected lane: expect `bytes` on the barrier, then start the copy global -> shared
__device__ __forceinline__ void bulk_load_row(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t mbar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t mbar, uint32_t parity) {
    uint32_t done = 0;
    do {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(mbar), "r"(parity) : "memory");
    } while (!done);
}

// distances of ids[0..n) -> dist[0..n), two per step (one per half-warp).
// STAGES == 0: each lane loads its float4s straight from HBM.  STAGES > 0: base vectors are brought into a per-warp ring
// of STAGES shared-memory slots by bulk asynchronous copies (one 16-byte-aligned contiguous row each), STAGES rows in
// flight per warp, so the HBM latency of the next rows hides behind the arithmetic of the current pair.
template <int METRIC, int STAGES>
__device__ __forceinline__ void batch_distances(const HnswDev& ix, const float* qs, const uint32_t* ids, float* dist,
                                                uint32_t n, int lane, float* ring, uint32_t mbar0, uint32_t& phase_bits) {
    const int half = lane >> 4, hl = lane & 15;
    if (STAGES == 0) {
        for (uint32_t b = 0; b < n; b += 2) {
            const uint32_t slot = b + half;
            const uint32_t node = ids[min(slot, n - 1)];
            const float d = half_warp_distance<METRIC, false>(ix, qs, ix.vec + static_cast<uint64_t>(node) * ix.vstride, hl);
            if (hl == 0 && slot < n) dist[slot] = d;
        }
        __syncwarp();
        return;
    }
    const uint32_t bytes = ix.vstride * 4u;
    const uint32_t ring0 = smem_addr(ring);
    if (lane == 0) {
        const uint32_t first = min(static_cast<uint32_t>(STAGES), n);
        for (uint32_t s = 0; s < first; ++s)
            bulk_load_row(ring0 + s * bytes, ix.vec + static_cast<uint64_t>(ids[s]) * ix.vstride, bytes, mbar0 + 8u * s);
    }
    for (uint32_t b = 0; b < n; b += 2) {
        constexpr uint32_t kRing = STAGES > 0 ? STAGES : 1;  // (STAGES == 0 never reaches this path)
        const uint32_t slot0 = b % kRing, slot1 = (b + 1) % kRing;
        const bool second = (b + 1) < n;
        const uint32_t my = (half && second) ? slot1 : slot0;
        mbar_wait(mbar0 + 8u * my, (phase_bits >> my) & 1u);
        const float d = half_warp_distance<METRIC, true>(ix, qs, ring + static_cast<size_t>(my) * ix.vstride, hl);
        if (hl == 0 && (b + half) < n) dist[b + half] = d;
        phase_bits ^= (1u << slot0) | (second ? (1u << slot1) : 0u);
        __syncwarp();  // both slots fully consumed before they are refilled
        if (lane == 0) {
            const uint32_t nxt = b + STAGES;
            if (nxt < n) bulk_load_row(ring0 + slot0 * bytes, ix.vec + static_cast<uint64_t>(ids[nxt]) * ix.vstride, bytes, mbar0 + 8u * slot0);
            if (nxt + 1 < n) bulk_load_row(ring0 + slot1 * bytes, ix.vec + static_cast<uint64_t>(ids[nxt + 1]) * ix.vstride, bytes, mbar0 + 8u * slot1);
        }
    }
    __syncwarp();
}

// ---- sparse rows: ordered intersection ---------------------------------------------------------------------------------
constexpr uint32_t kSpFilterWords = 256;  // 8,192-bit membership filter of the query row's indices, per warp
constexpr uint32_t kSpQcapMax = 4096;     // query entries staged per warp at most (longer rows are searched in global memory)

__device__ __forceinline__ uint32_t sp_hash(uint32_t idx) { return (idx * 2654435761u) >> 19; }  // 13 bits

struct SparseQuery {  // one query row: generic pointers (shared-memory copy, or the global arrays for very long rows)
    const uint32_t* idx;
    const float* val;
    uint32_t n;
    const uint32_t* filter;
    bool nonfinite;  // sparse "l2": the row stores a NaN or +-inf, so its squared norm in the reference is NaN
};

__device__ __forceinline__ uint2 ld_stream_u2(const uint2* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}

// one 16-entry step of a half-warp: look the lane's entry up, then add the matched products of this step in entry order
__device__ __forceinline__ float sparse_step(const SparseQuery& q, bool has, uint2 ent, float ret, int lane) {
    bool hit = false;
    float prod = 0.0f;
    if (has) {
        const uint32_t h = sp_hash(ent.x);
        if ((q.filter[h >> 5] >> (h & 31u)) & 1u) {
            uint32_t lo = 0, hi = q.n;  // std::lower_bound
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (q.idx[mid] < ent.x) lo = mid + 1; else hi = mid;
            }
            if (lo < q.n && q.idx[lo] == ent.x) { hit = true; prod = __fmul_rn(q.val[lo], __uint_as_float(ent.y)); }
        }
    }
    const unsigned m = __ballot_sync(kFull, hit);
    if (m == 0u) return ret;
    const int half = lane >> 4;
    unsigned mh = (m >> (16 * half)) & 0xFFFFu;
    const int n_it = max(__popc(m & 0xFFFFu), __popc(m >> 16));
    for (int it = 0; it < n_it; ++it) {
        const int src = mh ? (__ffs(mh) - 1 + 16 * half) : lane;
        const float pv = __shfl_sync(kFull, prod, src);
        if (mh) { ret = __fadd_rn(ret, pv); mh &= mh - 1u; }
    }
    return ret;
}

// distances of ids[0..n) -> dist[0..n) for a sparse index, two rows at a time (one per half-warp).  The reference's sparse "l2"
// adds the squared norms do_l2_distance_simd(x, x) + do_l2_distance_simd(y, y) before subtracting 2<x,y> (feat_vectors.hpp:
// 186-192): 0 for finite rows, NaN when either row stores a NaN or +-inf anywhere, matched or not.  So l2 reads every stored
// value, also for an empty query, and returns NaN for such a pair.
template <int METRIC>
__device__ __forceinline__ void batch_distances_sparse(const HnswDev& ix, const SparseQuery& q, const uint32_t* ids, float* dist,
                                                       uint32_t n, int lane, unsigned long long& n_entries) {
    const int half = lane >> 4, hl = lane & 15;
    for (uint32_t b = 0; b < n; b += 2) {
        const uint32_t slot = b + half;
        const bool valid = slot < n;
        unsigned long long r0 = 0, r1 = 0;
        if (valid) {
            const uint32_t node = ids[slot];
            r0 = ix.sp_ptr[node];
            r1 = ix.sp_ptr[node + 1];
        }
        const uint32_t len = static_cast<uint32_t>(r1 - r0);
        const uint32_t len_max = max(len, __shfl_xor_sync(kFull, len, 16));
        if (hl == 0) n_entries += len;
        const uint2* row = ix.sp_ent + r0;
        float ret = 0.0f;
        bool nonfinite = false;  // l2: a stored NaN or +-inf among this lane's entries of the row
        for (uint32_t j0 = 0; j0 < len_max; j0 += 64) {  // four independent 128-byte loads per half-warp in flight
            uint2 e[4];
            bool has[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const uint32_t j = j0 + 16u * u + hl;
                has[u] = (j < len) && (METRIC == HNSW_L2 || q.n != 0u);
                e[u] = has[u] ? ld_stream_u2(row + j) : make_uint2(0u, 0u);
                if (METRIC == HNSW_L2) nonfinite |= has[u] && !isfinite(__uint_as_float(e[u].y));
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                if (j0 + 16u * u < len_max) ret = sparse_step(q, has[u], e[u], ret, lane);
            }
        }
        float d = sparse_finalize<METRIC>(ret);
        if (METRIC == HNSW_L2) {
            const unsigned bad = (__ballot_sync(kFull, nonfinite) >> (16 * half)) & 0xFFFFu;
            if (bad || q.nonfinite) d = __uint_as_float(0x7FFFFFFFu);
        }
        if (hl == 0 && valid) dist[slot] = d;
    }
    __syncwarp();
}

// ---- libstdc++ heap algorithms (std::push_heap / std::pop_heap), entries {dist bits, node}; MAXH: std::less ---------
template <bool MAXH>
__device__ __forceinline__ bool heap_comp(uint2 a, float value_dist) {
    const float ad = __uint_as_float(a.x);
    return MAXH ? (ad < value_dist) : (ad > value_dist);
}

template <bool MAXH>
__device__ __forceinline__ void heap_sift_up(uint2* h, int hole, int top, uint2 value) {
    const float vd = __uint_as_float(value.x);
    int parent = (hole - 1) / 2;
    while (hole > top && heap_comp<MAXH>(h[parent], vd)) {
        h[hole] = h[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    h[hole] = value;
}

template <bool MAXH>
__device__ __forceinline__ void heap_adjust(uint2* h, int hole, int len, uint2 value) {
    const int top = hole;
    int child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (heap_comp<MAXH>(h[child], __uint_as_float(h[child - 1].x))) child--;
        h[hole] = h[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        h[hole] = h[child - 1];
        hole = child - 1;
    }
    heap_sift_up<MAXH>(h, hole, top, value);
}

template <bool MAXH>
__device__ __forceinline__ void heap_push(uint2* h, int& n, float dist, uint32_t node) {
    const uint2 v = make_uint2(__float_as_uint(dist), node);
    h[n] = v;
    ++n;
    heap_sift_up<MAXH>(h, n - 1, 0, v);
}

template <bool MAXH>
__device__ __forceinline__ void heap_pop(uint2* h, int& n) {
    if (n > 1) {
        const uint2 value = h[n - 1];
        h[n - 1] = h[0];
        heap_adjust<MAXH>(h, 0, n - 1, value);
    }
    --n;
}

__device__ __forceinline__ uint32_t permuted_pos_dev(const HnswDev& ix, uint32_t i) {
    const uint32_t m = (ix.feat_dim >> 4) << 4;
    if (i < m) {
        const uint32_t k = i >> 4, j = i & 15u;
        return 64u * (k >> 2) + 4u * j + (k & 3u);
    }
    return ix.main_pad + (i - m);
}

}  // namespace

}  // namespace pb200
