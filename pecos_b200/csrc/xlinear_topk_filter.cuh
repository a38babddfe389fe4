// xl_topk_filter_kernel: exact top-k of a query's candidate row with the expensive post-processor evaluated only for
// the few candidates that can possibly be selected.
//
// Included by xlinear_engine.cu (inside its anonymous namespace, after xl_transform / xl_combine / last_le_u32).
//
// The reference transforms EVERY candidate through double-precision exp/log/pow (pecos/core/xmc/inference.hpp:208-238,
// :1360-1384) and then selects k of them (:1223-1298).  On the GPU those double chains were ~85 % of the top-k kernel's
// instructions although only k of ~160..1,840 candidates survive.  Here:
//
//   pass 1  every candidate gets a cheap single-precision estimate s~ of its final score (|s~ - s| <= 1e-5 |s| + 1e-37,
//           see xl_transform_estimate), stored as a 4-byte orderable key in shared memory; each lane tracks the maximum
//           of its stride-32 subset;
//   bound   T = the kk-th largest of the 32 lane maxima.  kk different candidates have s~ >= T, hence the exact kk-th
//           largest score s* >= T - err(T), hence every candidate of the exact top-kk has s~ >= T - 2 err(T).  We keep
//           everything with s~ >= T - (1e-3 |T| + 1e-30): a margin 50x wider than the estimate's error bound.  A
//           non-finite T keeps everything;
//   exact   survivors (typically kk + a few) are evaluated with the same double-precision code as before, 32 per batch,
//           one per lane, and merged into a running, lane-distributed sorted top-32 by a bitonic network on the same
//           64-bit composite key (orderable(score) << 32 | ~position) the other top-k kernels use.  Saturated
//           post-processors (hinge == 1.0 for hundreds of candidates) simply produce more batches.
//
// The selected ids, their order (score desc, position asc) and the value bits are therefore those of xl_topk_warp_kernel;
// tests/test_xlinear_gpu.py runs both against the oracle.  Eligibility (host): k <= 32, beam <= kFltSlots, candidate row
// <= kFltKeysMax, hinge power <= 4.
#pragma once

constexpr int kFltWarps = 4;           // queries per CTA
constexpr int kFltSlots = 64;          // beam slots
constexpr uint32_t kFltKeysMax = 8192; // candidate row capacity
constexpr int kFltRing = 256;          // pending survivor positions (>= 31 + 128)

__host__ __device__ inline size_t flt_warp_bytes(uint32_t key_cap) {
    return (static_cast<size_t>(key_cap) * 4 + (kFltSlots + 1 + kFltSlots + kFltSlots) * 4 + kFltRing * 2 + 4 + 15) &
           ~static_cast<size_t>(15);
}

// single-precision estimate of xl_transform.  Relative error <= ~1e-5 wherever the exact value is a normal float,
// absolute error <= 1e-37 otherwise (ex2.approx flushes denormals).
__device__ __forceinline__ float xl_transform_estimate(float v, int kind, int p) {
    switch (kind) {
        case PP_SIGMOID: return __fdividef(1.0f, 1.0f + __expf(-v));
        case PP_LOG_SIGMOID: return v < -20.0f ? v : -log1pf(__expf(-v));  // -log(1+e^-v) = v - log(1+e^v)
        case PP_LP_HINGE:
        case PP_LOG_LP_HINGE: {
            const float z = fmaxf(0.0f, 1.0f - v);
            float t;
            switch (p) {
                case 0: t = 1.0f; break;
                case 1: t = z; break;
                case 2: t = z * z; break;
                case 3: t = (z * z) * z; break;
                default: { const float z2 = z * z; t = z2 * z2; } break;
            }
            return kind == PP_LP_HINGE ? __expf(-t) : -t;
        }
        default: return v;
    }
}

// inverse of orderable (shard_merge.cuh)
__device__ __forceinline__ float xl_from_orderable(uint32_t o) {
    return __uint_as_float((o & 0x80000000u) ? (o ^ 0x80000000u) : ~o);
}

__device__ __forceinline__ unsigned long long xl_umax64(unsigned long long a, unsigned long long b) { return a > b ? a : b; }
__device__ __forceinline__ unsigned long long xl_umin64(unsigned long long a, unsigned long long b) { return a < b ? a : b; }

// descending sort of one key per lane (bitonic network, 15 compare-exchange steps)
__device__ __forceinline__ unsigned long long xl_warp_sort_desc(unsigned long long key, int lane) {
#pragma unroll
    for (int k = 2; k <= 32; k <<= 1) {
#pragma unroll
        for (int j = k >> 1; j > 0; j >>= 1) {
            const unsigned long long o = __shfl_xor_sync(kFull, key, j);
            const bool desc = (lane & k) == 0;   // k == 32: every lane
            const bool lower = (lane & j) == 0;
            key = (lower == desc) ? xl_umax64(key, o) : xl_umin64(key, o);
        }
    }
    return key;
}

// lanes hold a bitonic sequence -> descending order (5 steps)
__device__ __forceinline__ unsigned long long xl_warp_bitonic_merge_desc(unsigned long long key, int lane) {
#pragma unroll
    for (int j = 16; j > 0; j >>= 1) {
        const unsigned long long o = __shfl_xor_sync(kFull, key, j);
        key = ((lane & j) == 0) ? xl_umax64(key, o) : xl_umin64(key, o);
    }
    return key;
}

__global__ void __launch_bounds__(kFltWarps * 32)
xl_topk_filter_kernel(const LayerDev L, const int pp_kind, const int pp_p, const int combine, const uint32_t k,
                      const uint32_t* __restrict__ beam_id, const float* __restrict__ beam_val,
                      const uint32_t* __restrict__ beam_cnt, const uint32_t beam_stride, const float* __restrict__ cand,
                      const uint64_t cand_stride_q, uint32_t* __restrict__ out_id, float* __restrict__ out_val,
                      uint32_t* __restrict__ out_cnt, const uint32_t out_stride, const uint32_t rows,
                      unsigned long long* stats, unsigned long long* __restrict__ out_key, const uint32_t key_cap) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const uint32_t q = blockIdx.x * kFltWarps + warp;
    if (q >= rows) return;
    unsigned char* slice = smem_raw + warp * flt_warp_bytes(key_cap);
    uint32_t* keys = reinterpret_cast<uint32_t*>(slice);           // [key_cap] estimate keys (0 = not a candidate here)
    uint32_t* s_base = keys + key_cap;                             // [kFltSlots + 1]
    uint32_t* s_colbeg = s_base + (kFltSlots + 1);                 // [kFltSlots]
    float* s_pval = reinterpret_cast<float*>(s_colbeg + kFltSlots);  // [kFltSlots]
    unsigned short* ring = reinterpret_cast<unsigned short*>(s_pval + kFltSlots);  // [kFltRing]

    // ---- beam slots: width / first column / parent score; candidate positions by a warp scan over the widths
    const uint32_t cnt = beam_cnt[q];
    uint32_t run = 0, owned = 0;
    for (uint32_t j0 = 0; j0 < cnt; j0 += 32) {
        const uint32_t j = j0 + lane;
        uint32_t w = 0, cb = 0xFFFFFFFFu;
        float pv = 0.0f;
        if (j < cnt) {
            const uint32_t p = beam_id[static_cast<uint64_t>(q) * beam_stride + j];
            const uint4 h = *reinterpret_cast<const uint4*>(&L.chunks[p]);  // {col_begin, n_cols, nnz_rows, has_bias}
            pv = beam_val[static_cast<uint64_t>(q) * beam_stride + j];
            w = h.y;
            cb = (h.w & kChunkAbsent) ? 0xFFFFFFFFu : h.x;  // absent: scored on another GPU (index sharding)
        }
        uint32_t incl = w;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t t = __shfl_up_sync(kFull, incl, d);
            if (lane >= d) incl += t;
        }
        uint32_t mine = (cb != 0xFFFFFFFFu) ? w : 0u;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) mine += __shfl_xor_sync(kFull, mine, d);
        if (j < cnt) {
            s_base[j + 1] = run + incl;
            s_colbeg[j] = cb;
            s_pval[j] = pv;
        }
        owned += mine;
        run += __shfl_sync(kFull, incl, 31);
    }
    if (lane == 0) s_base[0] = 0;
    __syncwarp();
    const uint32_t n_valid = run;
    const uint32_t kk = min(k, owned);
    if (lane == 0) {
        out_cnt[q] = kk;
        if (stats) atomicAdd(&stats[6], static_cast<unsigned long long>(kk));
    }
    if (n_valid == 0 || kk == 0) return;
    const float* cq = cand + static_cast<uint64_t>(q) * cand_stride_q;
    const uint32_t n_pad = (n_valid + 127u) & ~127u;  // <= key_cap (host rounds the capacity to 128)

    // ---- pass 1: estimates.  A lane visits positions lane, lane+32, ... in increasing order, so its slot index only
    // moves forward.
    uint32_t mx = 0, slot = 0;
    for (uint32_t i0 = lane; i0 < n_pad; i0 += 256) {
        float r[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) { const uint32_t i = i0 + 32u * u; r[u] = (i < n_valid) ? cq[i] : 0.0f; }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const uint32_t i = i0 + 32u * u;
            uint32_t key = 0;
            if (i < n_valid) {
                while (i >= s_base[slot + 1]) ++slot;  // s_base[cnt] == n_valid > i
                if (s_colbeg[slot] != 0xFFFFFFFFu) {
                    float s = xl_transform_estimate(r[u], pp_kind, pp_p);
                    if (combine) s = xl_combine(s, s_pval[slot], pp_kind);
                    key = max(orderable(s), 1u);
                }
            }
            if (i < n_pad) keys[i] = key;
            mx = max(mx, key);
        }
    }
    // ---- lower bound T of the kk-th largest estimate: the kk-th largest lane maximum
    uint32_t tkey = 0;
    {
        uint32_t m = mx;
        for (uint32_t r = 0; r < kk; ++r) {
            tkey = __reduce_max_sync(kFull, m);
            if (tkey == 0) break;  // fewer than kk non-empty lanes: keep everything
            const int w = __ffs(__ballot_sync(kFull, m == tkey)) - 1;
            if (lane == w) m = 0;
        }
    }
    uint32_t cut = 1;
    if (tkey != 0) {
        const float T = xl_from_orderable(tkey);
        if (isfinite(T)) cut = max(orderable(T - (1e-3f * fabsf(T) + 1e-30f)), 1u);
    }
    __syncwarp();

    // ---- survivors -> exact keys, 32 at a time, merged into the running top-32 (lane r holds the r-th best)
    unsigned long long best = 0ull;
    uint32_t pend = 0, head = 0;
    const uint32_t n_it = n_pad >> 7;
    const unsigned lt_mask = (1u << lane) - 1u;
    for (uint32_t it = 0; it <= n_it; ++it) {
        const bool last = (it == n_it);
        if (!last) {
            const uint4 kv = reinterpret_cast<const uint4*>(keys)[it * 32 + lane];
            const uint32_t b = (it << 7) + (static_cast<uint32_t>(lane) << 2);
            const bool p0 = kv.x >= cut, p1 = kv.y >= cut, p2 = kv.z >= cut, p3 = kv.w >= cut;
            if (__ballot_sync(kFull, p0 | p1 | p2 | p3)) {
                unsigned m;
                m = __ballot_sync(kFull, p0);
                if (p0) ring[(head + pend + __popc(m & lt_mask)) & (kFltRing - 1)] = static_cast<unsigned short>(b);
                pend += __popc(m);
                m = __ballot_sync(kFull, p1);
                if (p1) ring[(head + pend + __popc(m & lt_mask)) & (kFltRing - 1)] = static_cast<unsigned short>(b + 1);
                pend += __popc(m);
                m = __ballot_sync(kFull, p2);
                if (p2) ring[(head + pend + __popc(m & lt_mask)) & (kFltRing - 1)] = static_cast<unsigned short>(b + 2);
                pend += __popc(m);
                m = __ballot_sync(kFull, p3);
                if (p3) ring[(head + pend + __popc(m & lt_mask)) & (kFltRing - 1)] = static_cast<unsigned short>(b + 3);
                pend += __popc(m);
                __syncwarp();
            }
        }
        while (pend >= 32u || (last && pend > 0u)) {
            const uint32_t take = min(pend, 32u);
            unsigned long long key = 0ull;
            if (static_cast<uint32_t>(lane) < take) {
                const uint32_t pos = ring[(head + lane) & (kFltRing - 1)];
                const uint32_t j = static_cast<uint32_t>(last_le_u32(s_base, static_cast<int>(cnt), pos));
                float v = xl_transform(cq[pos], pp_kind, pp_p);
                if (combine) v = xl_combine(v, s_pval[j], pp_kind);
                key = xl_exact_key(v, pos);
            }
            head = (head + take) & (kFltRing - 1);
            pend -= take;
            __syncwarp();
            key = xl_warp_sort_desc(key, lane);
            const unsigned long long rev = __shfl_sync(kFull, key, 31 - lane);
            best = xl_warp_bitonic_merge_desc(xl_umax64(best, rev), lane);
        }
    }

    // ---- results: lane r writes rank r
    if (static_cast<uint32_t>(lane) < kk) {
        const uint32_t pos = xl_exact_key_pos(best);
        const uint32_t j = static_cast<uint32_t>(last_le_u32(s_base, static_cast<int>(cnt), pos));
        uint32_t label = s_colbeg[j] + (pos - s_base[j]);
        if (L.label_of_col) label = L.label_of_col[label];
        const uint64_t o = static_cast<uint64_t>(q) * out_stride + lane;
        out_id[o] = label;
        out_val[o] = xl_exact_key_value(best);
        if (out_key) out_key[o] = (best & 0xFFFFFFFF00000000ull) | static_cast<unsigned long long>(0xFFFFFFFFu - pos);
    }
}
