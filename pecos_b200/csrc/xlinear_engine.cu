// XR-Linear beam search on H100 (sm_90a): kernels + engine.  See xlinear_engine.h for the reference map.
//
// Per tree layer two kernels run over a tile of queries:
//
//   xl_chunk_scores_kernel   one CTA per query, one warp per beam slot (= one weight chunk).  The warp streams the
//                            chunk's sorted row-index list from HBM with 128-bit loads, intersects it with the query's
//                            sorted feature list held in shared memory, gathers the matched rows' {col,val} entries and
//                            accumulates them into the chunk's dense output block IN THE REFERENCE'S ORDER:
//                            ascending feature index, separate round-to-nearest multiply and add, bias row last
//                            (inference.hpp:788-811; dense queries: bias first, inference.hpp:823-837).
//                            HBM-bound; algorithmic bytes per (query, chunk) = 32 + 4R + 16m + 8e + 4c  (SURVEY 8d).
//
//   xl_topk_kernel           one CTA per query: post-processor transform in double precision (inference.hpp:208-238),
//                            combine with the parent's path score, then exact top-k on the composite key
//                            (score desc, position-in-prolongated-row asc) == sorted_csr's comparator
//                            (inference.hpp:1265-1273).  Bitonic sort of 64-bit keys in shared memory.
//
// No FMA contraction anywhere on the score path: products use __fmul_rn, sums use __fadd_rn (the reference build has
// no -march flag, so its XR-Linear loops are scalar mulss/addss).
#include "xlinear_engine.h"
#include "shard_merge.cuh"

#include <algorithm>
#include <atomic>
#include <cstring>
#include <exception>
#include <thread>

namespace pb200 {

namespace {

constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int kWarpsMax = 10;    // warps per CTA of the chunk kernel
constexpr int kMCap = 256;       // match list capacity per warp
constexpr int kMFlush = 128;     // flush the match list once it holds this many rows (kMCap - 128 new per pass)
constexpr int kCSmem = 128;      // chunk widths up to this accumulate in shared memory, wider ones in the HBM block
constexpr int kQCap = 1024;      // query non-zeros staged in shared memory (longer queries are read through L1/L2)
constexpr int kSortCap = 2048;   // keys sorted in shared memory per pass of the top-k kernel
constexpr int kTopkThreads = 256;

constexpr int kMCapLookup = 256; // the lookup kernel collects a block of <= 128 matches (+ bias row) between flush checks

template <int MCAP>
struct __align__(16) WarpScratch {
    uint32_t ms[MCAP];         // chunk-row index of each match; becomes the row's first entry offset during flush
    float mx[MCAP];            // multiplier of the row: query value, or the bias
    uint32_t off[MCAP + 4];    // exclusive prefix of the matched rows' entry counts
    float out[kCSmem];         // dense output block of the chunk
};

__device__ __forceinline__ uint4 ld_stream_u4(const uint32_t* p) {
    uint4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p));
    return r;
}

__device__ __forceinline__ int lower_bound_u32(const uint32_t* a, int n, uint32_t key) {
    int lo = 0, hi = n;
    while (lo < hi) {
        int mid = (lo + hi) >> 1;
        if (a[mid] < key) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// largest i in [0, n) with a[i] <= key, given a[0] <= key
__device__ __forceinline__ int last_le_u32(const uint32_t* a, int n, uint32_t key) {
    int lo = 0, hi = n;
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (a[mid] <= key) lo = mid; else hi = mid;
    }
    return lo;
}

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        uint32_t t = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v += t;
    }
    return v;
}

// Rows of the 32 consecutive entries [G, G + 32) of the concatenated matched rows (off[] = their prefix sums, off[m] =
// total, every row non-empty).  row_first = row holding entry G (warp-uniform; updated to the row holding entry G + 32).
// Lane L looks at candidate row row_first + 1 + L: if it starts inside the group it sets the bit of its first entry; a
// lane's row is then row_first + (number of row starts at or before the lane).  ~12 instructions instead of a
// log2(m)-step binary search per entry.
__device__ __forceinline__ int xl_rows_of_group(const uint32_t* off, int m, uint32_t G, int& row_first, int lane) {
    const int r = row_first + 1 + lane;
    uint32_t bit = 0;
    if (r < m) {
        const uint32_t p = off[r] - G;
        if (p < 32u) bit = 1u << p;
    }
    const uint32_t starts = __reduce_or_sync(kFull, bit);
    const int my_row = row_first + __popc(starts & (0xFFFFFFFFu >> (31 - lane)));
    const int r31 = __shfl_sync(kFull, my_row, 31);
    row_first = (off[r31 + 1] == G + 32u) ? r31 + 1 : r31;
    return my_row;
}

// Apply the matched rows collected in ws (in ascending feature order) to the output block.
//
// Entry-parallel: the m matched rows hold `total` entries; lane L of group g owns entry 32g + L of their concatenation
// (its row found by a binary search in the rows' prefix sums), so ragged rows -- one entry for a rare feature, every column
// for the bias row -- cost the same per entry, consecutive lanes read consecutive entries, and nothing is staged in
// shared memory.  Entries of one 32-group that hit the same column (they come from different rows, or from a row that
// repeats a column) are added in lane order = concatenation order = ascending feature order; __match_any_sync finds the
// collisions, so the common collision-free group costs a single round.  Groups are applied in order.
template <int MCAP>
__device__ __forceinline__ void xl_flush_impl(WarpScratch<MCAP>& ws, int m, const uint2* __restrict__ ext,
                                              const uint2* __restrict__ ent, float* out, int lane,
                                              unsigned long long& e_total) {
    if (m == 0) return;
    __syncwarp();
    constexpr int PER = MCAP / 32;
    uint32_t c[PER];
    uint32_t local = 0;
    bool empty_row = false;
#pragma unroll
    for (int u = 0; u < PER; ++u) {  // PER independent 8-byte loads per lane; ms[i]: chunk row -> its first entry
        const int i = lane * PER + u;
        c[u] = 0;
        if (i < m) {
            const uint2 lh = __ldg(ext + ws.ms[i]);
            ws.ms[i] = lh.x;
            c[u] = lh.y - lh.x;
            empty_row |= (c[u] == 0u);
        }
        local += c[u];
    }
    const bool search = __any_sync(kFull, empty_row);  // never for chunks built from a CSC matrix (rows have >= 1 entry)
    const uint32_t incl = warp_incl_scan(local, lane);
    uint32_t run = incl - local;
    const uint32_t total = __shfl_sync(kFull, incl, 31);
#pragma unroll
    for (int u = 0; u < PER; ++u) {
        const int i = lane * PER + u;
        if (i < m) { ws.off[i] = run; run += c[u]; }
    }
    if (lane == 0) ws.off[m] = total;
    __syncwarp();
    e_total += total;

    int row_first = 0;
    for (uint32_t g0 = 0; g0 < total; g0 += 128u) {
        uint2 e[4];
        float x[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {  // four entry loads in flight per lane
            const uint32_t G = g0 + 32u * u;
            const uint32_t g = G + lane;
            e[u] = make_uint2(0xFFFFFFFFu - lane, 0u);  // idle lanes: distinct pseudo-columns, never applied
            x[u] = 0.0f;
            if (G < total) {
                int i = 0;
                if (!search) i = xl_rows_of_group(ws.off, m, G, row_first, lane);
                if (g < total) {
                    if (search) i = last_le_u32(ws.off, m, g);  // off[i] <= g < off[i + 1]
                    e[u] = __ldg(ent + ws.ms[i] + (g - ws.off[i]));
                    x[u] = ws.mx[i];
                }
            }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            if (g0 + 32u * u >= total) break;
            const bool valid = (g0 + 32u * u + lane) < total;
            const float v = __fmul_rn(x[u], __uint_as_float(e[u].y));
            const unsigned peers = __match_any_sync(kFull, e[u].x);
            const uint32_t rank = __popc(peers & ((1u << lane) - 1u));
            const uint32_t rounds = __reduce_max_sync(kFull, valid ? rank : 0u);
            for (uint32_t r = 0; r <= rounds; ++r) {
                if (valid && rank == r) out[e[u].x] = __fadd_rn(out[e[u].x], v);
                __syncwarp();
            }
        }
    }
}

// out-of-line copy for the kernels that flush from several places
template <int MCAP>
__device__ __noinline__ void xl_flush(WarpScratch<MCAP>& ws, int m, const uint2* __restrict__ ext,
                                      const uint2* __restrict__ ent, float* out, int lane, unsigned long long& e_total) {
    xl_flush_impl(ws, m, ext, ent, out, lane, e_total);
}

// DENSE: row-major dense queries.  LOOKUP: sparse queries probe the chunk's feature map (one 8-byte cell per query
// feature) instead of streaming the chunk's row list -- same matches in the same order, far fewer bytes/instructions.
template <bool DENSE, bool STATS, bool LOOKUP>
__global__ void __launch_bounds__(kWarpsMax * 32, LOOKUP ? 4 : 1)  // lookup variant: <= 51 registers => 4 x 10-warp CTAs per SM
xl_chunk_scores_kernel(const LayerDev L, const QueryDev X, const uint32_t* __restrict__ beam_id,
                       const uint32_t* __restrict__ beam_cnt, const uint32_t beam_stride, float* __restrict__ cand,
                       const uint64_t cand_stride_q, const uint32_t c_stride, unsigned long long* stats,
                       const uint32_t q_cap, const uint32_t sb_cap, const uint32_t hdr_cap) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    uint32_t* q_idx_s = reinterpret_cast<uint32_t*>(smem_raw);
    float* q_val_s = reinterpret_cast<float*>(smem_raw + q_cap * 4);
    uint32_t* slot_base = reinterpret_cast<uint32_t*>(smem_raw + q_cap * 8);  // [cnt + 1] first candidate of each beam slot
    ChunkHeader* hdr_s = reinterpret_cast<ChunkHeader*>(smem_raw + q_cap * 8 + sb_cap * 4);  // [hdr_cap] beam chunk headers
    constexpr int MCAP = LOOKUP ? kMCapLookup : kMCap;
    WarpScratch<MCAP>* scratch =
        reinterpret_cast<WarpScratch<MCAP>*>(smem_raw + q_cap * 8 + sb_cap * 4 + static_cast<size_t>(hdr_cap) * sizeof(ChunkHeader));

    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int nwarps = blockDim.x >> 5;
    const uint32_t q = blockIdx.x;

    // ---- prologue.  All global loads are issued before the first shared-memory store (issue is in order: a store that
    // waits for its operand would otherwise serialise the independent load chains below).
    const uint32_t cnt = beam_cnt[q];
    uint64_t qb = 0, qe = 0;
    if (!DENSE) { qb = X.row_ptr[q] - X.nnz_base; qe = X.row_ptr[q + 1] - X.nnz_base; }
    const uint32_t my_p = (threadIdx.x < cnt) ? beam_id[static_cast<uint64_t>(q) * beam_stride + threadIdx.x] : 0u;
    const uint32_t* qidx = nullptr;
    const float* qval = nullptr;
    int qn = 0;
    uint32_t first_idx = 0;
    float first_val = 0.0f;
    bool staged = false;
    if (!DENSE) {
        qn = static_cast<int>(qe - qb);
        qidx = X.col_idx + qb;
        qval = X.val + qb;
        staged = qn <= static_cast<int>(q_cap);
        if (staged && static_cast<int>(threadIdx.x) < qn) { first_idx = qidx[threadIdx.x]; first_val = qval[threadIdx.x]; }
    } else {
        qval = X.val + static_cast<uint64_t>(q) * X.cols;
    }
    ChunkHeader my_h;
    my_h.n_cols = 0;
    if (threadIdx.x < cnt) my_h = L.chunks[my_p];
    if (staged) {
        if (static_cast<int>(threadIdx.x) < qn) { q_idx_s[threadIdx.x] = first_idx; q_val_s[threadIdx.x] = first_val; }
        for (int i = threadIdx.x + blockDim.x; i < qn; i += blockDim.x) { q_idx_s[i] = qidx[i]; q_val_s[i] = qval[i]; }
        qidx = q_idx_s;
        qval = q_val_s;
    }
    // candidates of a query are stored compactly in prolongation order: slot j starts at the sum of the widths before it
    if (threadIdx.x < cnt) {
        slot_base[threadIdx.x + 1] = my_h.n_cols;
        my_h.col_begin = my_p;  // this kernel never needs col_begin: the cached copy carries the chunk id instead
        if (threadIdx.x < hdr_cap) hdr_s[threadIdx.x] = my_h;
    }
    for (uint32_t j = threadIdx.x + blockDim.x; j < cnt; j += blockDim.x) {
        const uint32_t pj = beam_id[static_cast<uint64_t>(q) * beam_stride + j];
        ChunkHeader hh = L.chunks[pj];
        slot_base[j + 1] = hh.n_cols;
        hh.col_begin = pj;
        if (j < hdr_cap) hdr_s[j] = hh;
    }
    __syncthreads();
    if (warp == 0) {  // widths -> first candidate position of every slot (warp scan, 32 slots per step)
        uint32_t run = 0;
        for (uint32_t j0 = 0; j0 < cnt; j0 += 32) {
            const uint32_t j = j0 + lane;
            const uint32_t w = (j < cnt) ? slot_base[j + 1] : 0u;
            const uint32_t incl = warp_incl_scan(w, lane);
            if (j < cnt) slot_base[j + 1] = run + incl;
            run += __shfl_sync(kFull, incl, 31);
        }
        if (lane == 0) slot_base[0] = 0;
    }
    __syncthreads();
    WarpScratch<MCAP>& ws = scratch[warp];
    unsigned long long st_chunks = 0, st_rows = 0, st_match = 0, st_ent = 0, st_cols = 0;

    for (uint32_t j = warp; j < cnt; j += nwarps) {
        uint32_t p;
        ChunkHeader h;
        if (j < hdr_cap) {
            h = hdr_s[j];
            p = h.col_begin;
        } else {
            p = beam_id[static_cast<uint64_t>(q) * beam_stride + j];
            h = L.chunks[p];
        }
        if (h.has_bias & kChunkAbsent) continue;  // leaf chunk owned by another GPU (index sharding): not scored here
        const bool chunk_bias = (h.has_bias & 1u) != 0u;
        const uint32_t R = h.nnz_rows;
        const uint32_t R4 = (R + 3u) & ~3u;
        const uint32_t* ridx = L.meta + h.meta_off;
        const uint2* ext = reinterpret_cast<const uint2*>(L.rowext + h.meta_off);  // {begin, end} of every chunk row
        const uint2* ent = L.entries + h.ent_off;
        float* blk = cand + static_cast<uint64_t>(q) * cand_stride_q + slot_base[j];
        const bool in_smem = h.n_cols <= static_cast<uint32_t>(kCSmem);
        float* out = in_smem ? ws.out : blk;
        for (uint32_t c = lane; c < h.n_cols; c += 32) out[c] = 0.0f;
        __syncwarp();

        int m = 0;
        unsigned long long e_total = 0, m_total = 0;

        if (DENSE) {
            // chunk_ops<drm, bin_search>: bias row first, then every chunk row (inference.hpp:823-837)
            const uint32_t r_lim = chunk_bias ? R - 1u : R;
            if (chunk_bias) {
                if (lane == 0) { ws.ms[0] = R - 1u; ws.mx[0] = L.bias; }
                m = 1;
                __syncwarp();
            }
            for (uint32_t base = 0; base < r_lim; base += 128u) {
                const uint32_t i = base + lane * 4u;
                const uint32_t n_here = (i < r_lim) ? min(4u, r_lim - i) : 0u;
                uint4 v = make_uint4(0, 0, 0, 0);
                if (n_here) v = ld_stream_u4(ridx + i);
                const uint32_t incl = warp_incl_scan(n_here, lane);
                const uint32_t tot = __shfl_sync(kFull, incl, 31);
                uint32_t pos = m + incl - n_here;
                if (n_here > 0) { ws.ms[pos] = i; ws.mx[pos] = qval[v.x]; }
                if (n_here > 1) { ws.ms[pos + 1] = i + 1; ws.mx[pos + 1] = qval[v.y]; }
                if (n_here > 2) { ws.ms[pos + 2] = i + 2; ws.mx[pos + 2] = qval[v.z]; }
                if (n_here > 3) { ws.ms[pos + 3] = i + 3; ws.mx[pos + 3] = qval[v.w]; }
                m += static_cast<int>(tot);
                if (m >= kMFlush) {
                    m_total += m;
                    xl_flush(ws, m, ext, ent, out, lane, e_total);
                    m = 0;
                }
            }
        } else {
            // chunk_ops<csr, bin_search>: matched rows in ascending feature order, bias row last (inference.hpp:788-811)
            if (LOOKUP) {
                // Blocks of 128 query features: four probe rounds issued back to back (4 independent cell loads in flight
                // per lane), matches compacted in feature order.  The match list takes a whole block (+ the bias row), so
                // the single flush site sits outside the probe registers' live range.
                const uint2* fm = L.featmap + static_cast<uint64_t>(p) * L.fm_words;
                int tb0 = 0;
                do {
                    if (R > 0 && tb0 < qn) {
                        uint2 cell[4];
                        uint32_t feat[4];
                        bool live[4];
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            const int t = tb0 + 32 * u + lane;
                            live[u] = false;
                            feat[u] = 0;
                            cell[u] = make_uint2(0u, 0u);
                            if (t < qn) {
                                const uint32_t f = qidx[t];
                                // a repeated column index only counts once: the reference's marching loop consumes the first
                                const bool dup = (t > 0) && (qidx[t - 1] == f);
                                if (!dup && f < L.w_rows) { live[u] = true; feat[u] = f; cell[u] = __ldg(fm + (f >> 5)); }
                            }
                        }
#pragma unroll
                        for (int u = 0; u < 4; ++u) {
                            if (tb0 + 32 * u >= qn) break;
                            const int t = tb0 + 32 * u + lane;
                            const uint32_t bit = feat[u] & 31u;
                            const bool hit = live[u] && ((cell[u].x >> bit) & 1u);
                            const unsigned mask = __ballot_sync(kFull, hit);
                            if (mask == 0u) continue;
                            if (hit) {
                                const uint32_t pos = m + __popc(mask & ((1u << lane) - 1u));
                                ws.ms[pos] = cell[u].y + __popc(cell[u].x & ((1u << bit) - 1u));
                                ws.mx[pos] = qval[t];
                            }
                            m += __popc(mask);
                        }
                    }
                    tb0 += 128;
                    const bool last_block = tb0 >= qn;
                    if (last_block && chunk_bias) {
                        __syncwarp();
                        if (lane == 0) { ws.ms[m] = R - 1u; ws.mx[m] = L.bias; }
                        ++m;
                    }
                    if (last_block || m > MCAP - 130) {  // room for the next block of <= 128 matches and the bias row
                        m_total += m;
                        xl_flush_impl(ws, m, ext, ent, out, lane, e_total);
                        m = 0;
                    }
                } while (tb0 < qn);
            } else if (qn > 0 && R > 0) {
                const uint32_t qmin = qidx[0];
                const uint32_t qmax = qidx[qn - 1];
                const uint4 sentinel = make_uint4(0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu, 0xFFFFFFFFu);
                uint32_t i = lane * 4u;
                uint4 v_next = (i < R4) ? ld_stream_u4(ridx + i) : sentinel;
                for (uint32_t base = 0; base < R4; base += 128u) {
                    const uint4 v = v_next;
                    i = base + lane * 4u;
                    const uint32_t i_n = i + 128u;
                    v_next = (i_n < R4) ? ld_stream_u4(ridx + i_n) : sentinel;
                    const uint32_t first = __shfl_sync(kFull, v.x, 0);
                    if (first > qmax) break;  // the remaining (sorted) chunk rows lie beyond the query's last feature
                    int t0 = -1, t1 = -1, t2 = -1, t3 = -1;
                    if (v.x >= qmin && v.x <= qmax) { int t = lower_bound_u32(qidx, qn, v.x); if (t < qn && qidx[t] == v.x) t0 = t; }
                    if (v.y >= qmin && v.y <= qmax) { int t = lower_bound_u32(qidx, qn, v.y); if (t < qn && qidx[t] == v.y) t1 = t; }
                    if (v.z >= qmin && v.z <= qmax) { int t = lower_bound_u32(qidx, qn, v.z); if (t < qn && qidx[t] == v.z) t2 = t; }
                    if (v.w >= qmin && v.w <= qmax) { int t = lower_bound_u32(qidx, qn, v.w); if (t < qn && qidx[t] == v.w) t3 = t; }
                    const uint32_t n_here = (t0 >= 0) + (t1 >= 0) + (t2 >= 0) + (t3 >= 0);
                    if (__ballot_sync(kFull, n_here > 0) == 0u) continue;
                    const uint32_t incl = warp_incl_scan(n_here, lane);
                    const uint32_t tot = __shfl_sync(kFull, incl, 31);
                    uint32_t pos = m + incl - n_here;
                    if (t0 >= 0) { ws.ms[pos] = i; ws.mx[pos] = qval[t0]; ++pos; }
                    if (t1 >= 0) { ws.ms[pos] = i + 1; ws.mx[pos] = qval[t1]; ++pos; }
                    if (t2 >= 0) { ws.ms[pos] = i + 2; ws.mx[pos] = qval[t2]; ++pos; }
                    if (t3 >= 0) { ws.ms[pos] = i + 3; ws.mx[pos] = qval[t3]; ++pos; }
                    m += static_cast<int>(tot);
                    if (m >= kMFlush) {
                        m_total += m;
                        xl_flush(ws, m, ext, ent, out, lane, e_total);
                        m = 0;
                    }
                }
            }
            if (!LOOKUP && chunk_bias) {
                __syncwarp();
                if (lane == 0) { ws.ms[m] = R - 1u; ws.mx[m] = L.bias; }
                ++m;
            }
        }
        if (!LOOKUP || DENSE) {
            m_total += m;
            xl_flush(ws, m, ext, ent, out, lane, e_total);
        }
        __syncwarp();
        if (in_smem) {
            for (uint32_t c = lane; c < h.n_cols; c += 32) blk[c] = ws.out[c];
        }
        __syncwarp();
        if (STATS) { st_chunks += 1; st_rows += R; st_match += m_total; st_ent += e_total; st_cols += h.n_cols; }
    }
    if (STATS) {
        if (lane == 0 && st_chunks) {
            atomicAdd(&stats[0], st_chunks);
            atomicAdd(&stats[1], st_rows);
            atomicAdd(&stats[2], st_match);
            atomicAdd(&stats[3], st_ent);
            atomicAdd(&stats[4], st_cols);
        }
        if (threadIdx.x == 0 && cnt > 0) atomicAdd(&stats[5], static_cast<unsigned long long>(DENSE ? X.cols : qn));
    }
}

// ------------------------------------------------------------------------------------------------------------------
// post-processor (inference.hpp:208-238).  The reference evaluates these through double precision libm calls and
// narrows to float; we do the same arithmetic with CUDA's double routines.  exp/log may differ from glibc in the last
// ulp of the DOUBLE result, which survives the narrowing to float only with probability ~2^-29 per element.
// Integer powers p <= 4 are formed by exact/singly-rounded multiplications (== correctly rounded pow).
// ------------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double xl_hinge_pow(float v, int p) {
    const double zd = fmax(0.0, 1.0 - static_cast<double>(v));
    const float z = static_cast<float>(zd);
    const double x = static_cast<double>(z);
    switch (p) {
        case 0: return 1.0;
        case 1: return x;
        case 2: return x * x;
        case 3: return (x * x) * x;
        case 4: { const double x2 = x * x; return x2 * x2; }
        default: return pow(x, static_cast<double>(static_cast<size_t>(static_cast<long long>(p))));
    }
}

__device__ __forceinline__ float xl_transform(float v, int kind, int p) {
    switch (kind) {
        case PP_SIGMOID: {
            const float e = static_cast<float>(exp(static_cast<double>(-v)));  // expf(-v), correctly rounded
            return static_cast<float>(1.0 / (1.0 + static_cast<double>(e)));
        }
        case PP_LOG_SIGMOID: {
            const float e = static_cast<float>(exp(static_cast<double>(-v)));
            return static_cast<float>(-log(1.0 + static_cast<double>(e)));
        }
        case PP_LP_HINGE: return static_cast<float>(exp(-xl_hinge_pow(v, p)));
        case PP_LOG_LP_HINGE: return static_cast<float>(-xl_hinge_pow(v, p));
        default: return v;
    }
}

__device__ __forceinline__ float xl_combine(float x, float parent, int kind) {
    switch (kind) {
        case PP_SIGMOID:
        case PP_LP_HINGE: return __fmul_rn(x, parent);
        case PP_LOG_SIGMOID:
        case PP_LOG_LP_HINGE: return __fadd_rn(x, parent);
        default: return x;
    }
}

__device__ __forceinline__ unsigned long long xl_make_key(float v, uint32_t pos) {
    uint32_t u = __float_as_uint(v);
    if ((u & 0x7FFFFFFFu) == 0u) u = 0u;  // -0.0 and +0.0 compare equal in the reference comparator
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return (static_cast<unsigned long long>(u) << 32) | static_cast<unsigned long long>(0xFFFFFFFFu - pos);
}

// Selection key that also carries the value's exact bits: orderable(score) << 32 | ~((pos << 1) | neg_zero).  Same order as
// xl_make_key (-0.0 ties with +0.0, and ties go to the lower position); xl_exact_key_value gives back the bits, -0.0 included.
__device__ __forceinline__ unsigned long long xl_exact_key(float v, uint32_t pos) {
    uint32_t u = __float_as_uint(v);
    const uint32_t neg_zero = (u == 0x80000000u) ? 1u : 0u;  // -0.0 compares equal to +0.0 but keeps its bits
    if ((u & 0x7FFFFFFFu) == 0u) u = 0u;
    u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
    return (static_cast<unsigned long long>(u) << 32) | static_cast<unsigned long long>(0xFFFFFFFFu - ((pos << 1) | neg_zero));
}
__device__ __forceinline__ uint32_t xl_exact_key_pos(unsigned long long key) {
    return (0xFFFFFFFFu - static_cast<uint32_t>(key & 0xFFFFFFFFull)) >> 1;
}
__device__ __forceinline__ float xl_exact_key_value(unsigned long long key) {
    const uint32_t hi = static_cast<uint32_t>(key >> 32);
    const uint32_t bits = (hi & 0x80000000u) ? (hi ^ 0x80000000u) : ~hi;
    return __uint_as_float(((0xFFFFFFFFu - static_cast<uint32_t>(key & 0xFFFFFFFFull)) & 1u) ? 0x80000000u : bits);
}

#include "xlinear_qw_kernel.cuh"
#include "xlinear_cm_kernel.cuh"

// descending bitonic sort of n (power of two) keys; a may live in shared or global memory
__device__ void xl_bitonic_desc(unsigned long long* a, uint32_t n) {
    for (uint32_t k = 2; k <= n; k <<= 1) {
        for (uint32_t j = k >> 1; j > 0; j >>= 1) {
            for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
                const uint32_t ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long x = a[i], y = a[ixj];
                    const bool desc_block = ((i & k) == 0);
                    if (desc_block ? (x < y) : (x > y)) { a[i] = y; a[ixj] = x; }
                }
            }
            __syncthreads();
        }
    }
}

__device__ __forceinline__ uint32_t next_pow2_u32(uint32_t v) {
    if (v <= 2) return 2;
    return 1u << (32 - __clz(v - 1));
}

__global__ void __launch_bounds__(kTopkThreads)
xl_topk_kernel(const LayerDev L, const int pp_kind, const int pp_p, const int combine, const uint32_t k,
               const uint32_t* __restrict__ beam_id, const float* __restrict__ beam_val,
               const uint32_t* __restrict__ beam_cnt, const uint32_t beam_stride, const float* __restrict__ cand,
               const uint64_t cand_stride_q, const uint32_t c_stride, uint32_t* __restrict__ out_id,
               float* __restrict__ out_val, uint32_t* __restrict__ out_cnt, const uint32_t out_stride,
               unsigned long long* sortbuf, const uint64_t sortbuf_stride, const uint32_t b_prev,
               unsigned long long* stats, unsigned long long* __restrict__ out_key) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);
    uint32_t* s_base = reinterpret_cast<uint32_t*>(smem_raw + kSortCap * 8);  // [b_prev + 1]
    uint32_t* s_colbeg = s_base + (b_prev + 1);                               // [b_prev]
    float* s_pval = reinterpret_cast<float*>(s_colbeg + b_prev);              // [b_prev]

    const uint32_t q = blockIdx.x;
    const uint32_t cnt = beam_cnt[q];
    for (uint32_t j = threadIdx.x; j < cnt; j += blockDim.x) {
        const uint32_t p = beam_id[static_cast<uint64_t>(q) * beam_stride + j];
        const ChunkHeader h = L.chunks[p];
        s_base[j + 1] = h.n_cols;
        s_colbeg[j] = (h.has_bias & kChunkAbsent) ? 0xFFFFFFFFu : h.col_begin;  // absent: candidates exist elsewhere
        s_pval[j] = beam_val[static_cast<uint64_t>(q) * beam_stride + j];
    }
    __syncthreads();
    __shared__ uint32_t s_owned;
    if (threadIdx.x == 0) {
        uint32_t run = 0, owned = 0;
        s_base[0] = 0;
        for (uint32_t j = 0; j < cnt; ++j) {
            if (s_colbeg[j] != 0xFFFFFFFFu) owned += s_base[j + 1];
            run += s_base[j + 1];
            s_base[j + 1] = run;
        }
        s_owned = owned;
    }
    __syncthreads();
    const uint32_t n_valid = s_base[cnt];       // positions are global (all beam slots), keys only for owned slots
    const uint32_t kk = min(k, s_owned);
    if (threadIdx.x == 0) {
        out_cnt[q] = kk;
        if (stats) atomicAdd(&stats[6], static_cast<unsigned long long>(kk));
    }
    if (n_valid == 0) return;

    const float* cq = cand + static_cast<uint64_t>(q) * cand_stride_q;
    auto score_at = [&](uint32_t cpos, uint32_t& label) -> float {
        const uint32_t j = static_cast<uint32_t>(last_le_u32(s_base, static_cast<int>(cnt), cpos));
        const uint32_t off = cpos - s_base[j];
        float v = xl_transform(cq[cpos], pp_kind, pp_p);
        if (combine) v = xl_combine(v, s_pval[j], pp_kind);
        label = s_colbeg[j] + off;
        return v;
    };
    auto key_at = [&](uint32_t cpos) -> unsigned long long {
        const uint32_t j = static_cast<uint32_t>(last_le_u32(s_base, static_cast<int>(cnt), cpos));
        if (s_colbeg[j] == 0xFFFFFFFFu) return 0ull;  // scored on another GPU
        uint32_t lab;
        return xl_make_key(score_at(cpos, lab), cpos);
    };

    unsigned long long* sorted = keys;
    if (n_valid <= static_cast<uint32_t>(kSortCap)) {
        const uint32_t P = next_pow2_u32(n_valid);
        for (uint32_t i = threadIdx.x; i < P; i += blockDim.x) {
            unsigned long long key = 0ull;
            if (i < n_valid) key = key_at(i);
            keys[i] = key;
        }
        __syncthreads();
        xl_bitonic_desc(keys, P);
    } else if (k <= static_cast<uint32_t>(kSortCap / 2)) {
        // streaming: keys[0, KP) hold the best so far, keys[KP, kSortCap) the next tile of candidates
        const uint32_t KP = next_pow2_u32(k);
        const uint32_t tile = kSortCap - KP;
        for (uint32_t i = threadIdx.x; i < KP; i += blockDim.x) keys[i] = 0ull;
        for (uint32_t t0 = 0; t0 < n_valid; t0 += tile) {
            for (uint32_t i = threadIdx.x; i < tile; i += blockDim.x) {
                const uint32_t cpos = t0 + i;
                unsigned long long key = 0ull;
                if (cpos < n_valid) key = key_at(cpos);
                keys[KP + i] = key;
            }
            __syncthreads();
            xl_bitonic_desc(keys, kSortCap);
        }
    } else {
        // wide beam AND large k: sort the whole candidate list in the HBM scratch
        sorted = sortbuf + static_cast<uint64_t>(q) * sortbuf_stride;
        const uint32_t P = next_pow2_u32(n_valid);
        for (uint32_t i = threadIdx.x; i < P; i += blockDim.x) {
            unsigned long long key = 0ull;
            if (i < n_valid) key = key_at(i);
            sorted[i] = key;
        }
        __syncthreads();
        xl_bitonic_desc(sorted, P);
    }

    for (uint32_t r = threadIdx.x; r < kk; r += blockDim.x) {
        const uint32_t cpos = 0xFFFFFFFFu - static_cast<uint32_t>(sorted[r] & 0xFFFFFFFFull);
        uint32_t label;
        const float v = score_at(cpos, label);  // recomputed so that the stored value keeps its exact bits (-0.0)
        if (L.label_of_col) label = L.label_of_col[label];
        out_id[static_cast<uint64_t>(q) * out_stride + r] = label;
        out_val[static_cast<uint64_t>(q) * out_stride + r] = v;
        if (out_key) out_key[static_cast<uint64_t>(q) * out_stride + r] = sorted[r];
    }
}

// Narrow-beam variant: one WARP per query (kSelWarps queries per CTA).  The keys of the <= kSelKeys candidates sit in the
// warp's shared-memory slice; the top-k is extracted by k rounds of warp arg-max on the 64-bit composite key (keys are
// unique because they embed the candidate position), the winning lane rescanning only its own stride-32 subset.
// Same keys, same order, same values as xl_topk_kernel.  (kSelWarps queries per CTA: shard_merge.cuh.)
constexpr int kSelKeysMax = 4096; // warp top-k capacity (dynamic shared memory, sized per launch)
constexpr int kSelSlots = 64;
constexpr int kSelK = 64;

struct SelScratch {  // view into the warp's slice of dynamic shared memory
    unsigned long long* keys;
    uint32_t* base;    // [kSelSlots + 1]
    uint32_t* colbeg;  // [kSelSlots]
    float* pval;       // [kSelSlots]
};

__host__ __device__ inline size_t sel_warp_bytes(uint32_t key_cap) {
    return static_cast<size_t>(key_cap) * 8 + (kSelSlots + 1 + kSelSlots + kSelSlots) * 4 + 12;  // padded to 16 below
}

__global__ void __launch_bounds__(kSelWarps * 32)
xl_topk_warp_kernel(const LayerDev L, const int pp_kind, const int pp_p, const int combine, const uint32_t k,
                    const uint32_t* __restrict__ beam_id, const float* __restrict__ beam_val,
                    const uint32_t* __restrict__ beam_cnt, const uint32_t beam_stride, const float* __restrict__ cand,
                    const uint64_t cand_stride_q, const uint32_t c_stride, uint32_t* __restrict__ out_id,
                    float* __restrict__ out_val, uint32_t* __restrict__ out_cnt, const uint32_t out_stride,
                    const uint32_t rows, unsigned long long* stats, unsigned long long* __restrict__ out_key,
                    const uint32_t key_cap) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const uint32_t q = blockIdx.x * kSelWarps + warp;
    if (q >= rows) return;
    const size_t slice = (sel_warp_bytes(key_cap) + 15) & ~static_cast<size_t>(15);
    SelScratch S;
    S.keys = reinterpret_cast<unsigned long long*>(smem_raw + warp * slice);
    S.base = reinterpret_cast<uint32_t*>(S.keys + key_cap);
    S.colbeg = S.base + (kSelSlots + 1);
    S.pval = reinterpret_cast<float*>(S.colbeg + kSelSlots);
    const uint32_t cnt = beam_cnt[q];
    for (uint32_t j = lane; j < cnt; j += 32) {
        const uint32_t p = beam_id[static_cast<uint64_t>(q) * beam_stride + j];
        const ChunkHeader h = L.chunks[p];
        S.base[j + 1] = h.n_cols;
        S.colbeg[j] = (h.has_bias & kChunkAbsent) ? 0xFFFFFFFFu : h.col_begin;
        S.pval[j] = beam_val[static_cast<uint64_t>(q) * beam_stride + j];
    }
    __syncwarp();
    uint32_t owned = 0;
    if (lane == 0) {
        uint32_t run = 0;
        S.base[0] = 0;
        for (uint32_t j = 0; j < cnt; ++j) {
            if (S.colbeg[j] != 0xFFFFFFFFu) owned += S.base[j + 1];
            run += S.base[j + 1];
            S.base[j + 1] = run;
        }
    }
    owned = __shfl_sync(kFull, owned, 0);
    __syncwarp();
    const uint32_t n_valid = S.base[cnt];
    const uint32_t kk = min(k, owned);
    if (lane == 0) {
        out_cnt[q] = kk;
        if (stats) atomicAdd(&stats[6], static_cast<unsigned long long>(kk));
    }
    if (n_valid == 0) return;
    const float* cq = cand + static_cast<uint64_t>(q) * cand_stride_q;
    auto score_at = [&](uint32_t cpos, uint32_t& label) -> float {
        const uint32_t j = static_cast<uint32_t>(last_le_u32(S.base, static_cast<int>(cnt), cpos));
        const uint32_t off = cpos - S.base[j];
        float v = xl_transform(cq[cpos], pp_kind, pp_p);
        if (combine) v = xl_combine(v, S.pval[j], pp_kind);
        label = S.colbeg[j] + off;
        return v;
    };
    // pass 1: raw scores -> shared memory; the candidates of a query are contiguous, so this is a flat coalesced copy
    // with eight independent loads in flight per lane
    for (uint32_t i0 = lane; i0 < n_valid; i0 += 256) {
        float r[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) { const uint32_t i = i0 + 32u * u; r[u] = (i < n_valid) ? cq[i] : 0.0f; }
#pragma unroll
        for (int u = 0; u < 8; ++u) { const uint32_t i = i0 + 32u * u; if (i < n_valid) S.keys[i] = static_cast<unsigned long long>(__float_as_uint(r[u])); }
    }
    __syncwarp();
    if (owned != n_valid) {  // index sharding: the ranges of leaf chunks scored on other GPUs hold no data
        for (uint32_t j = 0; j < cnt; ++j) {
            if (S.colbeg[j] != 0xFFFFFFFFu) continue;
            for (uint32_t i = S.base[j] + lane; i < S.base[j + 1]; i += 32) S.keys[i] = 0xFFFFFFFFFFFFFFFFull;
        }
        __syncwarp();
    }
    // pass 2: post-processor (double-precision libm chains), combine, composite key.  Four independent candidates per lane
    // and step, so the long dependent exp/log chains of different candidates overlap.
    for (uint32_t i0 = lane; i0 < n_valid; i0 += 128) {
        unsigned long long raw[4];
        float pv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const uint32_t i = i0 + 32u * u;
            raw[u] = 0xFFFFFFFFFFFFFFFFull;
            pv[u] = 0.0f;
            if (i < n_valid) {
                raw[u] = S.keys[i];
                pv[u] = S.pval[last_le_u32(S.base, static_cast<int>(cnt), i)];
            }
        }
        float v[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) v[u] = xl_transform(__uint_as_float(static_cast<uint32_t>(raw[u])), pp_kind, pp_p);
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const uint32_t i = i0 + 32u * u;
            if (i < n_valid) {
                float w = v[u];
                if (combine) w = xl_combine(w, pv[u], pp_kind);
                S.keys[i] = (raw[u] == 0xFFFFFFFFFFFFFFFFull) ? 0ull : xl_make_key(w, i);
            }
        }
    }
    __syncwarp();
    unsigned long long best = 0ull;  // lane-local maximum over positions lane, lane+32, ...
    for (uint32_t i = lane; i < n_valid; i += 32) { const unsigned long long key = S.keys[i]; best = key > best ? key : best; }
    __syncwarp();
    for (uint32_t r = 0; r < kk; ++r) {
        unsigned long long top = best;
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            const unsigned long long o = __shfl_xor_sync(kFull, top, d);
            top = o > top ? o : top;
        }
        const uint32_t cpos = 0xFFFFFFFFu - static_cast<uint32_t>(top & 0xFFFFFFFFull);
        if ((cpos & 31u) == static_cast<uint32_t>(lane)) {
            uint32_t label;
            const float v = score_at(cpos, label);  // recomputed: keeps the exact bits (-0.0) of the stored value
            if (L.label_of_col) label = L.label_of_col[label];
            out_id[static_cast<uint64_t>(q) * out_stride + r] = label;
            out_val[static_cast<uint64_t>(q) * out_stride + r] = v;
            if (out_key) out_key[static_cast<uint64_t>(q) * out_stride + r] = top;
            S.keys[cpos] = 0ull;
            best = 0ull;
            for (uint32_t i = lane; i < n_valid; i += 32) { const unsigned long long key = S.keys[i]; best = key > best ? key : best; }
        }
        __syncwarp();
    }
}

#include "xlinear_topk_filter.cuh"

// predict_selected: one CTA per query; its entries [ent_ptr[q], ent_ptr[q + 1]) read candidate ent_pos[e] of the query's row
// and, when `combine`, the value of entry prev_ptr[q] + ent_parent[e] of the previous layer
__global__ void __launch_bounds__(128)
xl_selected_gather_kernel(const float* __restrict__ cand, const uint64_t cand_stride_q, const uint64_t* __restrict__ ent_ptr,
                          const uint32_t* __restrict__ ent_pos, const uint32_t* __restrict__ ent_parent,
                          const uint64_t* __restrict__ prev_ptr, const float* __restrict__ prev_val, float* __restrict__ cur_val,
                          const int pp_kind, const int pp_p, const int combine) {
    const uint32_t q = blockIdx.x;
    const uint64_t b = ent_ptr[q], e = ent_ptr[q + 1];
    const float* cq = cand + static_cast<uint64_t>(q) * cand_stride_q;
    const uint64_t pb = combine ? prev_ptr[q] : 0;
    for (uint64_t i = b + threadIdx.x; i < e; i += blockDim.x) {
        float v = xl_transform(cq[ent_pos[i]], pp_kind, pp_p);
        if (combine) v = xl_combine(v, prev_val[pb + ent_parent[i]], pp_kind);
        cur_val[i] = v;
    }
}

// Packed exchange records for index sharding (ShardRecord, shard_merge.cuh): ONE record per (query, rank) slot, key == 0
// marks an empty slot (a valid key is never 0: its low word is ~position), so the per-query counts need not travel: the
// whole exchange is a single all-gather of one buffer.
__global__ void xl_shard_pack_kernel(const unsigned long long* __restrict__ keys, const uint32_t* __restrict__ ids,
                                     const float* __restrict__ vals, const uint32_t* __restrict__ cnt, const uint32_t rows,
                                     const uint32_t stride, ShardRecord* __restrict__ rec) {
    const uint64_t i = static_cast<uint64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= static_cast<uint64_t>(rows) * stride) return;
    const uint32_t q = static_cast<uint32_t>(i / stride), r = static_cast<uint32_t>(i - static_cast<uint64_t>(q) * stride);
    ShardRecord out{0ull, 0u, 0.0f};
    if (r < cnt[q]) { out.key = keys[i]; out.id = ids[i]; out.val = vals[i]; }
    rec[i] = out;
}

// Row extents as one 8-byte record per chunk row, derived on the device from the row_ptr array of the chunk (the score
// kernels then need ONE load per matched row).  The chunk's region of meta[] holds R4 + roundup4(R + 1) >= 2R words, so
// rowext[] simply mirrors meta[]'s indexing.
__global__ void xl_build_rowext_kernel(const ChunkHeader* __restrict__ chunks, const uint32_t* __restrict__ meta,
                                       uint32_t* __restrict__ rowext, const uint32_t n_chunks) {
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (uint32_t c = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; c < n_chunks; c += warps) {
        const ChunkHeader h = chunks[c];
        if (h.has_bias & kChunkAbsent) continue;
        const uint32_t R = h.nnz_rows;
        const uint32_t* rp = meta + h.meta_off + ((R + 3u) & ~3u);
        uint2* dst = reinterpret_cast<uint2*>(rowext + h.meta_off);
        for (uint32_t r = lane; r < R; r += 32) dst[r] = make_uint2(rp[r], rp[r + 1]);
    }
}

__global__ void xl_init_beam_kernel(uint32_t* beam_id, float* beam_val, uint32_t* beam_cnt, uint32_t beam_stride,
                                    uint32_t rows) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q < rows) {
        beam_id[static_cast<uint64_t>(q) * beam_stride] = 0u;   // prev_layer_pred = ones(Q x 1) (inference.hpp:2462-2463)
        beam_val[static_cast<uint64_t>(q) * beam_stride] = 1.0f;
        beam_cnt[q] = 1u;
    }
}

uint32_t max_row_nnz(const uint64_t* row_ptr, uint32_t rows) {
    uint64_t m = 0;
    for (uint32_t r = 0; r < rows; ++r) m = std::max<uint64_t>(m, row_ptr[r + 1] - row_ptr[r]);
    return static_cast<uint32_t>(std::min<uint64_t>(m, 0xFFFFFFFFull));
}

uint32_t next_pow2_host(uint64_t v) {
    uint64_t p = 2;
    while (p < v) p <<= 1;
    return static_cast<uint32_t>(p);
}

size_t chunk_kernel_smem(int warps, bool lookup, uint32_t q_cap, uint32_t sb_cap, uint32_t hdr_cap) {
    return static_cast<size_t>(q_cap) * 8 + static_cast<size_t>(sb_cap) * 4 + static_cast<size_t>(hdr_cap) * sizeof(ChunkHeader) +
           static_cast<size_t>(warps) * (lookup ? sizeof(WarpScratch<kMCapLookup>) : sizeof(WarpScratch<kMCap>));
}
size_t topk_kernel_smem(uint32_t b_prev) { return static_cast<size_t>(kSortCap) * 8 + (static_cast<size_t>(b_prev) * 3 + 1) * 4; }
static_assert(kSortCap * 8 + (kXlBeamMaxTopk * 3 + 1) * 4 <= 200 * 1024 && kSortCap * 8 + ((kXlBeamMaxTopk + 1) * 3 + 1) * 4 > 200 * 1024,
              "kXlBeamMaxTopk is the widest beam whose block top-k fits 200 KB of shared memory");

// Widths of the beams entering each layer (the b_prev / k_cap chain of make_plan_); false at the first one over `limit`.
// k_last: the last layer's k_cap when every beam fits.
bool beam_chain_fits(const XLinearHostModel& m, uint32_t beam_size, uint32_t only_topk, const std::vector<uint32_t>& b_in,
                     uint32_t limit, uint32_t* layer, uint32_t* width, uint32_t* k_last = nullptr) {
    const size_t depth = m.layers.size();
    uint32_t b_prev = 1;
    for (size_t d = 0; d < depth; ++d) {
        const auto& L = m.layers[d];
        if (d < b_in.size() && b_in[d] > 0) b_prev = b_in[d];
        if (b_prev > limit) {
            if (layer) *layer = static_cast<uint32_t>(d);
            if (width) *width = b_prev;
            return false;
        }
        const uint32_t local = (d + 1 == depth) ? only_topk : beam_size;
        const uint32_t k = local > 0 ? local : static_cast<uint32_t>(L.only_topk);
        const uint64_t cand_max = static_cast<uint64_t>(b_prev) * std::max<uint32_t>(L.c_max, 1u);
        b_prev = static_cast<uint32_t>(std::max<uint64_t>(1, std::min<uint64_t>(k, cand_max)));
    }
    if (k_last) *k_last = b_prev;
    return true;
}

}  // namespace

uint32_t xlinear_plan_stride(const XLinearHostModel& m, uint32_t beam_size, uint32_t only_topk) {
    uint32_t k_last = 1;
    beam_chain_fits(m, beam_size, only_topk, {}, 0xFFFFFFFFu, nullptr, nullptr, &k_last);
    return k_last;
}

XLinearBeamCheck xlinear_check_beam(const XLinearHostModel& m, uint32_t beam_size, uint32_t only_topk,
                                    const std::vector<uint32_t>& b_in, bool topk) {
    XLinearBeamCheck r;
    r.limit = topk ? kXlBeamMaxTopk : kXlBeamMax;
    r.fits = beam_chain_fits(m, beam_size, only_topk, b_in, r.limit, &r.layer, &r.b_prev);
    // a wider beam_size never narrows a beam, so the plans that fit are the beam sizes up to some bound
    if (beam_chain_fits(m, 0xFFFFFFFFu, only_topk, b_in, r.limit, nullptr, nullptr)) {
        r.widest = 0xFFFFFFFFu;
    } else {
        uint32_t lo = 0, hi = 0xFFFFFFFFu;  // fits(lo) (or lo == 0), !fits(hi)
        while (hi - lo > 1) {
            const uint32_t mid = lo + (hi - lo) / 2;
            if (beam_chain_fits(m, mid, only_topk, b_in, r.limit, nullptr, nullptr)) lo = mid; else hi = mid;
        }
        r.widest = lo;
    }
    return r;
}

// ------------------------------------------------------------------------------------------------------------------
// engine
// ------------------------------------------------------------------------------------------------------------------
XLinearEngine::XLinearEngine(std::unique_ptr<XLinearHostModel> host, int device) : host_(std::move(host)), device_(device) {
    PB200_CUDA(cudaSetDevice(device_));
    PB200_CUDA(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
    for (auto& e : ev_) PB200_CUDA(cudaEventCreate(&e));
    PB200_CUDA(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));
    for (auto& s : stage_) {
        PB200_CUDA(cudaEventCreateWithFlags(&s.landed, cudaEventDisableTiming));
        PB200_CUDA(cudaEventCreateWithFlags(&s.consumed, cudaEventDisableTiming));
    }
    layers_.resize(host_->layers.size());
    uint64_t cmimg_budget = 8ull << 30;     // bytes of HBM the chunk images of the chunk-major kernel may take in total
    if (const char* env = std::getenv("PB200_CMIMG_MB")) cmimg_budget = std::strtoull(env, nullptr, 10) << 20;
    {
        int sms = 0;
        PB200_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device_));
        n_sm_ = static_cast<uint32_t>(std::max(sms, 1));
    }
    uint64_t featmap_budget = 32ull << 30;  // bytes of HBM the feature maps may take in total
    if (const char* env = std::getenv("PB200_FEATMAP_MB")) featmap_budget = std::strtoull(env, nullptr, 10) << 20;
    for (size_t d = 0; d < layers_.size(); ++d) {
        auto& src = host_->layers[d];
        auto& dst = layers_[d];
        upload_store_(src, dst);
        // query-driven lookup structure, unless it would blow the memory budget (then the kernel streams the row lists)
        if (featmap_budget >= feature_map_bytes(src)) {
            featmap_budget -= feature_map_bytes(src);
            build_feature_map(src);
            dst.featmap.upload(reinterpret_cast<const uint2*>(src.featmap.data()), src.featmap.size(), stream_);
            PB200_CUDA(cudaStreamSynchronize(stream_));
            dst.view.featmap = dst.featmap.get();
            dst.view.fm_words = src.fm_words;
            model_bytes_ += src.featmap.size() * 8;
            std::vector<uint2_host>().swap(src.featmap);
        }
        dst.rowext.reserve(std::max<uint64_t>(src.meta.size(), 4));
        xl_build_rowext_kernel<<<n_sm_ * 8, 256, 0, stream_>>>(dst.chunks.get(), dst.meta.get(), dst.rowext.get(), src.n_chunks);
        PB200_CUDA(cudaGetLastError());
        dst.view.rowext = dst.rowext.get();
        model_bytes_ += src.meta.size() * 4;
        // chunk images for the chunk-major score kernel (xlinear_cm_kernel.cuh), where the layer's shape allows it
        if (dst.view.featmap) {
            const CmLayout cm = cm_layer_layout(src);
            const uint64_t bytes = static_cast<uint64_t>(cm.shape.img_bytes) * cm.shape.n_vc;
            if (cm.shape.ok && bytes <= cmimg_budget) {
                cmimg_budget -= bytes;
                place_images_(dst, cm.shape, cm.vc_ptr);
            }
        }
    }
    // The prefix image: layers 0 and 1 merged into one chunk (build_prefix_layer) whose image has a direct table.
    if (layers_.size() >= 2 && layers_[0].view.featmap && layers_[1].view.featmap &&
        prefix_mergeable(host_->layers[0], host_->layers[1])) {
        ChunkedLayerHost M;
        build_prefix_layer(host_->layers[0], host_->layers[1], M);
        const uint32_t fm_words = static_cast<uint32_t>((static_cast<uint64_t>(M.w_rows) + 31) / 32);
        const uint64_t n_ent = M.entries.size();
        const CmShape shape = n_ent < 65535u ? cm_shape(fm_words, M.w_rows, M.r_max, static_cast<uint32_t>(n_ent), M.c_max, 1, 1) : CmShape{};
        if (shape.ok && shape.direct && shape.img_bytes <= cmimg_budget) {
            upload_store_(M, prefix_);
            place_images_(prefix_, shape, {0u, 1u});
            model_bytes_ += 2 * sizeof(uint32_t);  // model_bytes() counts the prefix's virtual-chunk table, not the layers'
            PB200_CUDA(cudaStreamSynchronize(stream_));  // M's host arrays go out of scope
        }
    }
    PB200_CUDA(cudaStreamSynchronize(stream_));
    // host copies of the big arrays are no longer needed
    for (auto& l : host_->layers) {
        std::vector<uint32_t>().swap(l.meta);
        std::vector<ChunkEntry>().swap(l.entries);
    }
    const int max_smem = 200 * 1024;
    PB200_CUDA(cudaFuncSetAttribute(xl_chunk_scores_kernel<false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(xl_chunk_scores_kernel<false, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(xl_chunk_scores_kernel<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(xl_chunk_scores_kernel<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(xl_chunk_scores_kernel<true, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(xl_chunk_scores_kernel<true, true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(xl_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(xl_topk_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(xl_topk_filter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(xl_cm_scores_kernel<true, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kCmSmemBudget)));
    PB200_CUDA(cudaFuncSetAttribute(xl_cm_scores_kernel<true, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kCmSmemBudget)));
    PB200_CUDA(cudaFuncSetAttribute(xl_cm_scores_kernel<false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kCmSmemBudget)));
    PB200_CUDA(cudaFuncSetAttribute(xl_cm_scores_kernel<false, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kCmSmemBudget)));
    PB200_CUDA(cudaFuncSetAttribute(xl_cm_scores_kernel<true, 2, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kCmSmemBudget)));
    PB200_CUDA(cudaFuncSetAttribute(xl_cm_scores_kernel<true, 4, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kCmSmemBudget)));
    PB200_CUDA(cudaFuncSetAttribute(xl_query_warp_scores_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    PB200_CUDA(cudaFuncSetAttribute(xl_query_warp_scores_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    stats_dev_.reserve(8 * layers_.size());
    if (const char* env = std::getenv("PB200_XL_KERNEL_MODE")) set_kernel_mode(std::atoi(env));  // A/B runs of bench.py
    layer_profile_.assign(layers_.size(), XLinearLayerProfile{});
    layer_stats_.assign(layers_.size(), XLinearStats{});
}

void XLinearEngine::upload_store_(const ChunkedLayerHost& H, LayerStore& S) {
    S.chunks.upload(H.chunks.data(), H.chunks.size(), stream_);
    S.meta.upload(H.meta.data(), H.meta.size(), stream_);
    S.entries.upload(reinterpret_cast<const uint2*>(H.entries.data()), H.entries.size(), stream_);
    if (H.reordered) S.label_of_col.upload(H.label_of_col.data(), H.label_of_col.size(), stream_);
    S.view.chunks = S.chunks.get();
    S.view.meta = S.meta.get();
    S.view.entries = S.entries.get();
    S.view.label_of_col = H.reordered ? S.label_of_col.get() : nullptr;
    S.view.n_cols = H.n_cols;
    S.view.n_chunks = H.n_chunks;
    S.view.c_max = H.c_max;
    S.view.w_rows = H.w_rows;
    S.view.bias = H.bias;
    model_bytes_ += H.chunks.size() * sizeof(ChunkHeader) + H.meta.size() * 4 + H.entries.size() * 8 + H.label_of_col.size() * 4;
}

void XLinearEngine::place_images_(LayerStore& S, CmShape shape, const std::vector<uint32_t>& vc_ptr) {
    S.cm_vc_ptr.upload(vc_ptr.data(), vc_ptr.size(), stream_);
    PB200_CUDA(cudaStreamSynchronize(stream_));  // the host table may go out of scope
    shape.vc_ptr = S.cm_vc_ptr.get();
    const uint64_t bytes = static_cast<uint64_t>(shape.img_bytes) * shape.n_vc;
    S.cm_images.reserve(bytes);
    xl_cm_build_images_kernel<<<shape.n_vc, 256, 0, stream_>>>(S.view, shape, S.cm_images.get());
    PB200_CUDA(cudaGetLastError());
    S.cm_shape = shape;
    model_bytes_ += bytes;
}

XLinearEngine::~XLinearEngine() {
    cudaSetDevice(device_);
    if (stream_) cudaStreamSynchronize(stream_);
    for (auto& e : ev_) if (e) cudaEventDestroy(e);
    if (copy_stream_) cudaStreamSynchronize(copy_stream_);
    for (auto& s : stage_) for (cudaEvent_t e : {s.landed, s.consumed}) if (e) cudaEventDestroy(e);
    if (copy_stream_) cudaStreamDestroy(copy_stream_);
    if (stream_) cudaStreamDestroy(stream_);
}

bool XLinearEngine::has_feature_maps() const {
    for (auto& l : layers_) if (!l.view.featmap) return false;
    return true;
}

void XLinearEngine::reset_profile() {
    layer_profile_.assign(layers_.size(), XLinearLayerProfile{});
    launches_ = 0;
}

std::vector<XLinearEngine::LayerPlan> XLinearEngine::make_plan_(uint32_t beam_size, const char* post_processor, uint32_t only_topk,
                                                                 const std::vector<uint32_t>& b_in, bool topk) const {
    const XLinearBeamCheck fit = xlinear_check_beam(*host_, beam_size, only_topk, b_in, topk);
    if (!fit.fits)
        throw std::runtime_error("pecos_b200: beam of " + std::to_string(fit.b_prev) + " nodes entering layer " +
                                 std::to_string(fit.layer) + " exceeds the supported maximum of " + std::to_string(fit.limit));
    const size_t depth = layers_.size();
    std::vector<LayerPlan> plan(depth);
    uint32_t b_prev = 1;
    for (size_t d = 0; d < depth; ++d) {
        const auto& L = host_->layers[d];
        if (d < b_in.size() && b_in[d] > 0) b_prev = b_in[d];
        // local_only_topk (inference.hpp:2471) then only_topk_to_use (inference.hpp:2055)
        const uint32_t local = (d + 1 == depth) ? only_topk : beam_size;
        const uint32_t k = local > 0 ? local : static_cast<uint32_t>(L.only_topk);
        plan[d].k = k;
        plan[d].pp = post_processor ? parse_post_processor(post_processor) : L.post_processor;
        plan[d].b_prev = b_prev;
        const uint64_t cand_max = static_cast<uint64_t>(b_prev) * std::max<uint32_t>(L.c_max, 1u);
        plan[d].k_cap = static_cast<uint32_t>(std::max<uint64_t>(1, std::min<uint64_t>(k, cand_max)));
        b_prev = plan[d].k_cap;
    }
    return plan;
}

uint32_t XLinearEngine::ensure_workspace_(const std::vector<LayerPlan>& plan, uint32_t rows, uint32_t dense_cols) {
    // per query: the two ping-pong beams (stride = the widest beam entering or leaving a layer), the candidate row, the sort
    // scratch of the block top-k, and the chunk-major kernel's slot positions and pair lists
    uint64_t beam_stride = 1, cand_max = 1, sort_max = 0, b_max = 1, chunks_max = 1;
    for (size_t d = 0; d < plan.size(); ++d) {
        const uint64_t c = static_cast<uint64_t>(plan[d].b_prev) * std::max<uint32_t>(host_->layers[d].c_max, 1u);
        cand_max = std::max(cand_max, c);
        beam_stride = std::max<uint64_t>(beam_stride, std::max<uint32_t>(plan[d].k_cap, plan[d].b_prev));
        if (c > static_cast<uint64_t>(kSortCap) && plan[d].k > static_cast<uint32_t>(kSortCap / 2)) sort_max = std::max<uint64_t>(sort_max, next_pow2_host(c));
        b_max = std::max<uint64_t>(b_max, plan[d].b_prev);
        chunks_max = std::max<uint64_t>(chunks_max, host_->layers[d].n_chunks);
    }
    const bool cm = chunk_major_workspace_();
    const uint64_t pairs = b_max * 4;  // up to 4 column ranges per chunk
    const uint64_t per_query = 16 + 2 * beam_stride * 8 + cand_max * 4 + sort_max * 8 + (cm ? beam_stride * 4 + pairs * 8 : 0);
    uint64_t budget = 8ull << 30;
    if (const char* env = std::getenv("PB200_WORKSPACE_MB")) budget = std::max<uint64_t>(64, std::strtoull(env, nullptr, 10)) << 20;
    uint64_t tile = std::min<uint64_t>(std::max<uint64_t>(1, budget / per_query), std::max<uint32_t>(rows, 1u));
    if (dense_cols) tile = std::min<uint64_t>(tile, std::max<uint64_t>(1, (4ull << 30) / (static_cast<uint64_t>(dense_cols) * 4)));

    beam_stride_ = static_cast<uint32_t>(beam_stride);
    for (int b = 0; b < 2; ++b) {
        beam_id_[b].reserve(tile * beam_stride);
        beam_val_[b].reserve(tile * beam_stride);
        beam_cnt_[b].reserve(tile);
    }
    if (cm) {
        cm_slot_pos_.reserve(tile * beam_stride);
        cm_pair_q_.reserve(tile * pairs);
        cm_pair_pos_.reserve(tile * pairs);
        cm_count_.reserve(chunks_max * 4 + 1);
        cm_claim_.reserve(chunks_max * 4 + 1);
        cm_active_.reserve(chunks_max * 4 + 1);
        cm_bucket_ptr_.reserve(chunks_max * 4 + 1);
        cm_cost_ptr_.reserve(chunks_max * 4 + 1);
    }
    cand_.reserve(tile * cand_max);
    if (sort_max) sortbuf_.reserve(tile * sort_max);
    return static_cast<uint32_t>(tile);
}

// Kernel ids, as XLinearLayerProfile and pb200_xlinear_get_kernel_ids report them.
enum : int { kScoreRowList = 0, kScoreLookup = 1, kScoreDense = 2, kScoreQueryWarp = 3, kScoreChunkMajor = 4 };
enum : int { kNoTopk = -1, kTopkBlock = 0, kTopkWarp = 1, kTopkFilter = 2 };

struct XLinearEngine::TileShape {  // run_tile_'s arguments; topk = false: no top-k kernel follows the scores (selected outputs)
    bool ext_beam;
    int combine_first;
    size_t d_begin, d_end;
    bool collect_stats, topk;
};

struct XLinearEngine::LayerKernels {
    int score = kScoreRowList;
    CmPlan cm;            // launch shape of the chunk-major score kernel (score == kScoreChunkMajor without the prefix)
    int topk = kNoTopk;   // kNoTopk: no top-k kernel runs, and the layer's reported top-k id keeps its last value
    bool prefix = false;  // layers 0 and 1 of the tile are scored by one prefix launch, issued at layer 0
};

// Chooses the kernels of layer d for one tile, from the kernel mode, the model and the call alone.
//
// Kernel modes (set_kernel_mode, PB200_XL_KERNEL_MODE), all with the same results: 0 first generation (every layer treated
// as having no feature map, block top-k); 1 default; 2 no query-warp kernel; 3 the query-warp kernel wherever it fits;
// 4 no estimate filter (the warp select evaluates every candidate); 5 the chunk-major kernel wherever a layer has images,
// and the prefix launch on tiles of any size (tests); 6 query-major kernels only (no chunk-major, no prefix); 7 no prefix.
//
// Order of preference [reported id]: score prefix [4] > chunk-major [4] > query-warp [3] > dense [2] > lookup [1] >
// row-list [0]; top-k filter [2] > warp select [1] > block sort [0], none for selected outputs nor for layer 0 under the
// prefix.  Candidate limits compare b_prev x c_max, the widest row the beam can produce.
XLinearEngine::LayerKernels XLinearEngine::pick_kernels_(size_t d, const QueryDev& q, const std::vector<LayerPlan>& plan,
                                                         const TileShape& t) const {
    const LayerStore& S = layers_[d];
    const LayerPlan& lp = plan[d];
    const uint64_t cand_stride_q = static_cast<uint64_t>(lp.b_prev) * std::max<uint32_t>(S.view.c_max, 1u);
    const bool sparse = q.row_ptr != nullptr;
    const bool first_gen = mode_ == KernelMode::kFirstGeneration;
    const bool force_cm = mode_ == KernelMode::kChunkMajorWherever;
    const bool cm_offsets_fit = static_cast<uint64_t>(q.rows) * std::max<uint32_t>(q.max_row_nnz, 1u) < (1ull << 32);  // 32-bit feature offsets
    LayerKernels k;

    // The prefix image exists only where layers 0 and 1 have feature maps.  Layer 0's top-k must keep all of layer 0, so that
    // layer 1's beam is all of layer 1 in layer 0's rank order.  A small tile leaves most SMs idle in the one-pass kernel,
    // while the per-layer kernels spread its pairs wider.
    const bool root_tile = !t.ext_beam && t.d_begin == 0 && t.d_end >= 2 && t.combine_first == 0 && !t.collect_stats;
    const bool prefix_mode = !first_gen && mode_ != KernelMode::kQueryMajorOnly && mode_ != KernelMode::kNoPrefix;
    const bool keeps_layer0 = plan[0].k >= host_->layers[0].n_cols;
    const bool fills_gpu = force_cm || q.rows >= kCmMinPairsPerSm * n_sm_;
    k.prefix = d < 2 && root_tile && prefix_mode && prefix_.cm_shape.ok && sparse && keeps_layer0 && cm_offsets_fit && fills_gpu;

    const bool lookup = sparse && !first_gen && S.view.featmap;  // mode 0: as if no layer had a feature map
    // the statistics pass runs the query-major kernels: their counters are the canonical ones
    if (!k.prefix && lookup && !t.collect_stats && cm_offsets_fit && chunk_major_workspace_())
        k.cm = cm_plan(S.cm_shape, S.view.n_chunks, static_cast<uint64_t>(q.rows) * lp.b_prev, n_sm_, force_cm);
    // One warp per query over the whole beam (feature-major) wins when the beam consists of MANY NARROW chunks (per-chunk
    // bookkeeping dominates: S layers 1-4, 20 x 8 columns), and loses on wide chunks where one warp per chunk keeps more
    // loads in flight (E and S leaves).
    const bool qw_fits = lookup && lp.b_prev <= static_cast<uint32_t>(kQwSlots) &&
                         cand_stride_q <= static_cast<uint64_t>(kQwNCap) && q.max_row_nnz <= kQwQCap;
    const bool query_warp = qw_fits && mode_ != KernelMode::kNoQueryWarp &&
                            (mode_ == KernelMode::kQueryWarpWherever || (lp.b_prev >= 16u && cand_stride_q <= 256u));
    k.score = (k.prefix || k.cm.eligible) ? kScoreChunkMajor : query_warp ? kScoreQueryWarp : !sparse ? kScoreDense
                                                             : lookup ? kScoreLookup : kScoreRowList;

    if (!t.topk || (k.prefix && d == 0)) return k;  // layer 0's beam comes out of the prefix launch
    const bool hinge = lp.pp.kind == PP_LP_HINGE || lp.pp.kind == PP_LOG_LP_HINGE;
    const bool exact_power = !hinge || (lp.pp.p >= 0 && lp.pp.p <= 4);  // the filter forms hinge powers up to 4 exactly
    const bool filter = !first_gen && mode_ != KernelMode::kNoTopkFilter && lp.k <= 32u && exact_power &&
                        lp.b_prev <= static_cast<uint32_t>(kFltSlots) && cand_stride_q <= static_cast<uint64_t>(kFltKeysMax);
    const bool warp_select = !first_gen && lp.b_prev <= static_cast<uint32_t>(kSelSlots) &&
                             cand_stride_q <= static_cast<uint64_t>(kSelKeysMax) && lp.k <= static_cast<uint32_t>(kSelK);
    k.topk = filter ? kTopkFilter : warp_select ? kTopkWarp : kTopkBlock;
    return k;
}

// Launches the score kernel k chose for layer d over the beam held in beam_*_[cur] (capacity b_prev slots per query): fills
// cand_[(ws_row + q) * b_prev * c_max + slot_base(j) + c] with the raw scores of every child of every beam node, in
// prolongation order.  Under the prefix, layer 0's launch also scores layer 1, and layer 1 launches nothing.
void XLinearEngine::score_layer_(size_t d, const QueryDev& q, const std::vector<LayerPlan>& plan, const LayerKernels& k, int cur,
                                 uint32_t ws_row, bool collect_stats) {
    layer_profile_[d].scores_kernel = k.score;
    if (k.prefix) {
        if (d == 0) launch_prefix_(q, plan, ws_row);
        return;
    }
    const LayerDev& L = layers_[d].view;
    const uint32_t b_prev = plan[d].b_prev;
    const uint32_t rows = q.rows;
    const bool dense = (q.row_ptr == nullptr);
    const uint32_t c_stride = std::max<uint32_t>(L.c_max, 1u);
    const uint64_t cand_stride_q = static_cast<uint64_t>(b_prev) * c_stride;
    float* cand = cand_.get() + ws_row * cand_stride_q;
    const uint32_t* bid = bid_(cur, ws_row);
    const uint32_t* bcnt = bcnt_(cur, ws_row);
    unsigned long long* stats = collect_stats ? stats_dev_.get() + 8 * d : nullptr;
    // spread the beam slots evenly: b = 10 -> 10 warps x 1 slot, b = 20 -> 10 warps x 2 slots
    const uint32_t rounds = (b_prev + kWarpsMax - 1) / kWarpsMax;
    const int warps = static_cast<int>(std::max<uint32_t>(1, (b_prev + rounds - 1) / std::max<uint32_t>(rounds, 1)));
    const dim3 grid(rows), block(warps * 32);
    const bool lookup = k.score == kScoreLookup;
    // query staging area: as small as the batch's longest row allows (occupancy), at most kQCap non-zeros
    const uint32_t q_cap = dense ? 32u : std::min<uint32_t>(kQCap, std::max<uint32_t>(32u, (q.max_row_nnz + 31u) & ~31u));
    const uint32_t sb_cap = (b_prev + 1u + 3u) & ~3u;
    const uint32_t hdr_cap = b_prev <= 128u ? b_prev : 0u;  // beam chunk headers cached in shared memory
    const size_t smem1 = chunk_kernel_smem(warps, lookup, q_cap, sb_cap, hdr_cap);
    auto launch = [&](auto kernel) {
        kernel<<<grid, block, smem1, stream_>>>(L, q, bid, bcnt, beam_stride_, cand,
                                               cand_stride_q, c_stride, stats, q_cap, sb_cap, hdr_cap);
    };
    if (k.score == kScoreChunkMajor) {
        const CmPlan& cm = k.cm;
        const CmShape& shape = layers_[d].cm_shape;
        const uint32_t n_vc = shape.n_vc;
        CmWork w{cm_slot_pos_.get(), cm_count_.get(), cm_bucket_ptr_.get(), cm_cost_ptr_.get(), cm_pair_q_.get(), cm_pair_pos_.get(),
                 cm_claim_.get(), cm_active_.get()};
        PB200_CUDA(cudaMemsetAsync(w.count, 0, (static_cast<uint64_t>(n_vc) + 1) * 4, stream_));
        const uint32_t bucket_grid = cm_bucket_grid(rows, n_sm_);
        xl_cm_count_kernel<<<bucket_grid, kCmBucketThreads, 0, stream_>>>(L, bid, bcnt, beam_stride_, rows, w, shape.vc_ptr, n_vc);
        xl_cm_scan_kernel<<<1, 1024, 0, stream_>>>(n_vc, w, layers_[d].cm_images.get(), shape.img_bytes, L.w_rows);
        xl_cm_scatter_kernel<<<bucket_grid, kCmBucketThreads, 0, stream_>>>(L, bid, bcnt, beam_stride_, rows, w, shape.vc_ptr, n_vc);
        auto launch_cm = [&](auto kernel) {
            kernel<<<cm.grid, cm.warps * 32, cm.smem, stream_>>>(L, q, w, shape, layers_[d].cm_images.get(), cand, cand_stride_q,
                                                                 CmPrefixOut{});
        };
        if (shape.direct) { if (shape.stages == 4) launch_cm(xl_cm_scores_kernel<true, 4>); else launch_cm(xl_cm_scores_kernel<true, 2>); }
        else { if (shape.stages == 4) launch_cm(xl_cm_scores_kernel<false, 4>); else launch_cm(xl_cm_scores_kernel<false, 2>); }
        launches_ += 3;  // + the score kernel counted below
    } else if (k.score == kScoreQueryWarp) {
        const uint32_t qw_qcap = std::max<uint32_t>(32u, (q.max_row_nnz + 31u) & ~31u);
        const uint32_t qw_ncap = static_cast<uint32_t>((cand_stride_q + 31) & ~static_cast<uint64_t>(31));
        const size_t qw_smem = kQwWarps * ((qw_warp_bytes(qw_qcap, qw_ncap) + 15) & ~static_cast<size_t>(15));
        const dim3 qw_grid((rows + kQwWarps - 1) / kQwWarps);
        if (collect_stats)
            xl_query_warp_scores_kernel<true><<<qw_grid, kQwWarps * 32, qw_smem, stream_>>>(
                L, q, bid, bcnt, beam_stride_, cand, cand_stride_q, stats, qw_qcap, qw_ncap, rows);
        else
            xl_query_warp_scores_kernel<false><<<qw_grid, kQwWarps * 32, qw_smem, stream_>>>(
                L, q, bid, bcnt, beam_stride_, cand, cand_stride_q, stats, qw_qcap, qw_ncap, rows);
    } else if (k.score == kScoreDense) {
        if (collect_stats) launch(xl_chunk_scores_kernel<true, true, false>);
        else launch(xl_chunk_scores_kernel<true, false, false>);
    } else if (lookup) {
        if (collect_stats) launch(xl_chunk_scores_kernel<false, true, true>);
        else launch(xl_chunk_scores_kernel<false, false, true>);
    } else {
        if (collect_stats) launch(xl_chunk_scores_kernel<false, true, false>);
        else launch(xl_chunk_scores_kernel<false, false, false>);
    }
    PB200_CUDA(cudaGetLastError());
    ++launches_;
}

void XLinearEngine::launch_prefix_(const QueryDev& q, const std::vector<LayerPlan>& plan, uint32_t ws_row) {
    const CmShape& S = prefix_.cm_shape;
    const uint32_t rows = q.rows;
    const uint32_t grid = std::min<uint32_t>(n_sm_, (rows + 31u) / 32u);
    const uint32_t share = (rows + grid - 1) / grid;
    const uint32_t warps = std::max<uint32_t>(1u, std::min<uint32_t>(S.warps_fit, (share + 31u) / 32u));
    const size_t smem = S.img_bytes + warps * cm_warp_bytes(S.acc_cols, S.stages) + 64;
    CmPrefixOut P;
    P.rows = rows;
    P.n0 = host_->layers[0].n_cols;
    P.pp_kind = plan[0].pp.kind;
    P.pp_p = plan[0].pp.p;
    P.chunks1 = layers_[1].view.chunks;
    P.beam_id = bid_(1, ws_row);
    P.beam_val = bval_(1, ws_row);
    P.beam_cnt = bcnt_(1, ws_row);
    P.beam_stride = beam_stride_;
    P.cand1_stride = static_cast<uint64_t>(plan[1].b_prev) * std::max<uint32_t>(layers_[1].view.c_max, 1u);
    P.cand1 = cand_.get() + ws_row * P.cand1_stride;
    auto launch = [&](auto kernel) {
        kernel<<<grid, warps * 32, smem, stream_>>>(prefix_.view, q, CmWork{}, S, prefix_.cm_images.get(), nullptr, 0, P);
    };
    if (S.stages == 4) launch(xl_cm_scores_kernel<true, 4, true>);
    else launch(xl_cm_scores_kernel<true, 2, true>);
    PB200_CUDA(cudaGetLastError());
    ++launches_;
}

// Runs layers [d_begin, d_end) over one tile of queries; the last layer of the plan writes into `out`.
void XLinearEngine::run_tile_(const QueryDev& q, const std::vector<LayerPlan>& plan, const OutTarget& out, uint32_t ws_row,
                              bool collect_stats, bool ext_beam, int combine_first, size_t d_begin, size_t d_end) {
    const uint32_t rows = q.rows;
    if (rows == 0) return;
    int cur = static_cast<int>(d_begin & 1);  // every layer flips the ping-pong beam buffers once
    const size_t depth = plan.size();
    d_end = std::min(d_end, depth);
    const TileShape t{ext_beam, combine_first, d_begin, d_end, collect_stats, true};
    for (size_t d = d_begin; d < d_end; ++d) {
        const LayerKernels k = pick_kernels_(d, q, plan, t);
        if (d == 0 && !ext_beam && !k.prefix) {  // the root beam (the prefix launch writes layer 0's beam itself)
            xl_init_beam_kernel<<<(rows + 255) / 256, 256, 0, stream_>>>(bid_(cur, ws_row), bval_(cur, ws_row),
                                                                         bcnt_(cur, ws_row), beam_stride_, rows);
            ++launches_;
        }
        if (profile_) PB200_CUDA(cudaEventRecord(ev_[0], stream_));
        score_layer_(d, q, plan, k, cur, ws_row, collect_stats);
        if (profile_) PB200_CUDA(cudaEventRecord(ev_[1], stream_));
        if (k.topk != kNoTopk) {
            const LayerDev& L = layers_[d].view;
            const LayerPlan& lp = plan[d];
            const int combine = (d == 0) ? combine_first : 1;
            const uint32_t c_stride = std::max<uint32_t>(L.c_max, 1u);
            const uint64_t cand_stride_q = static_cast<uint64_t>(lp.b_prev) * c_stride;
            const float* cand = cand_.get() + ws_row * cand_stride_q;
            const uint32_t* bid = bid_(cur, ws_row);
            const float* bval = bval_(cur, ws_row);
            const uint32_t* bcnt = bcnt_(cur, ws_row);
            unsigned long long* stats = collect_stats ? stats_dev_.get() + 8 * d : nullptr;
            const OutTarget o = (d + 1 == depth) ? out
                                                 : OutTarget{bid_(cur ^ 1, ws_row), bval_(cur ^ 1, ws_row), bcnt_(cur ^ 1, ws_row),
                                                             nullptr, beam_stride_};
            if (k.topk == kTopkFilter) {
                const uint32_t key_cap = static_cast<uint32_t>((cand_stride_q + 127) & ~static_cast<uint64_t>(127));
                const size_t flt_smem = kFltWarps * flt_warp_bytes(key_cap);
                xl_topk_filter_kernel<<<(rows + kFltWarps - 1) / kFltWarps, kFltWarps * 32, flt_smem, stream_>>>(
                    L, lp.pp.kind, lp.pp.p, combine, lp.k, bid, bval, bcnt,
                    beam_stride_, cand, cand_stride_q, o.ids, o.vals, o.cnt, o.stride, rows, stats, o.keys, key_cap);
            } else if (k.topk == kTopkWarp) {
                const uint32_t key_cap = static_cast<uint32_t>((cand_stride_q + 31) & ~static_cast<uint64_t>(31));
                const size_t sel_smem = kSelWarps * ((sel_warp_bytes(key_cap) + 15) & ~static_cast<size_t>(15));
                xl_topk_warp_kernel<<<(rows + kSelWarps - 1) / kSelWarps, kSelWarps * 32, sel_smem, stream_>>>(
                    L, lp.pp.kind, lp.pp.p, combine, lp.k, bid, bval, bcnt,
                    beam_stride_, cand, cand_stride_q, c_stride, o.ids, o.vals, o.cnt, o.stride, rows, stats, o.keys, key_cap);
            } else {
                xl_topk_kernel<<<rows, kTopkThreads, topk_kernel_smem(lp.b_prev), stream_>>>(
                    L, lp.pp.kind, lp.pp.p, combine, lp.k, bid, bval, bcnt,
                    beam_stride_, cand, cand_stride_q, c_stride, o.ids, o.vals, o.cnt, o.stride, sortbuf_.get(),
                    next_pow2_host(cand_stride_q), lp.b_prev, stats, o.keys);
            }
            PB200_CUDA(cudaGetLastError());
            ++launches_;
            layer_profile_[d].topk_kernel = k.topk;
        }
        if (profile_) {
            PB200_CUDA(cudaEventRecord(ev_[2], stream_));
            PB200_CUDA(cudaEventSynchronize(ev_[2]));
            float a = 0.f, b = 0.f;
            PB200_CUDA(cudaEventElapsedTime(&a, ev_[0], ev_[1]));
            PB200_CUDA(cudaEventElapsedTime(&b, ev_[1], ev_[2]));
            XLinearLayerProfile& p = layer_profile_[d];
            // under the prefix, layer 1's score slot stays at 0 ms (the launch is layer 0's), and layer 0's top-k slot too
            if (!(k.prefix && d == 1)) { p.scores_ms += a; ++p.launches; }
            if (k.topk != kNoTopk) { p.topk_ms += b; ++p.launches; }
        }
        cur ^= 1;
    }
}

XLinearEngine::Result XLinearEngine::finish_result_(const ResultBuffers& res, uint32_t rows, uint32_t stride) {
    out_ids_.reserve(static_cast<uint64_t>(rows) * stride + 1);
    out_vals_.reserve(static_cast<uint64_t>(rows) * stride + 1);
    out_cnt_.reserve(static_cast<uint64_t>(rows) + 1);
    if (rows) {
        PB200_CUDA(cudaMemcpyAsync(out_ids_.get(), res.ids.get(), static_cast<uint64_t>(rows) * stride * 4, cudaMemcpyDeviceToHost, stream_));
        PB200_CUDA(cudaMemcpyAsync(out_vals_.get(), res.vals.get(), static_cast<uint64_t>(rows) * stride * 4, cudaMemcpyDeviceToHost, stream_));
        PB200_CUDA(cudaMemcpyAsync(out_cnt_.get(), res.cnt.get(), static_cast<uint64_t>(rows) * 4, cudaMemcpyDeviceToHost, stream_));
    }
    PB200_CUDA(cudaStreamSynchronize(stream_));
    Result r;
    r.rows = rows;
    r.stride = stride;
    r.out_cols = host_->layers.back().out_cols;
    r.ids = out_ids_.get();
    r.vals = out_vals_.get();
    r.cnt = out_cnt_.get();
    return r;
}

XLinearEngine::OutTarget XLinearEngine::reserve_results_(ResultBuffers& res, uint32_t rows, uint32_t stride) {
    res.ids.reserve(static_cast<uint64_t>(rows) * stride + 1);
    res.vals.reserve(static_cast<uint64_t>(rows) * stride + 1);
    res.cnt.reserve(static_cast<uint64_t>(rows) + 1);
    return OutTarget{res.ids.get(), res.vals.get(), res.cnt.get(), nullptr, stride};
}

void XLinearEngine::QueryStage::reserve(const HostMatrix& x, uint32_t rows, uint64_t n) {
    if (!x.dense) {
        row_ptr.reserve(static_cast<uint64_t>(rows) + 1);
        col_idx.reserve(n);
    }
    val.reserve(n);
}

QueryDev XLinearEngine::QueryStage::place(const HostMatrix& x, uint32_t first, uint32_t r0, uint32_t tr, cudaStream_t stream) {
    if (x.dense) {
        const uint64_t n = static_cast<uint64_t>(tr) * x.cols;
        if (n) PB200_CUDA(cudaMemcpyAsync(val.get() + static_cast<uint64_t>(r0 - first) * x.cols, x.dense + static_cast<uint64_t>(r0) * x.cols,
                                          n * 4, cudaMemcpyHostToDevice, stream));
    } else {
        const uint64_t base = x.row_ptr[first], b = x.row_ptr[r0] - base, n = x.row_ptr[r0 + tr] - base - b;
        PB200_CUDA(cudaMemcpyAsync(row_ptr.get() + (r0 - first), x.row_ptr + r0, (static_cast<uint64_t>(tr) + 1) * 8, cudaMemcpyHostToDevice, stream));
        if (n) {
            PB200_CUDA(cudaMemcpyAsync(col_idx.get() + b, x.col_idx + base + b, n * 4, cudaMemcpyHostToDevice, stream));
            PB200_CUDA(cudaMemcpyAsync(val.get() + b, x.val + base + b, n * 4, cudaMemcpyHostToDevice, stream));
        }
    }
    return view(x, first, r0, tr);
}

QueryDev XLinearEngine::QueryStage::view(const HostMatrix& x, uint32_t first, uint32_t r0, uint32_t tr) const {
    if (x.dense) return QueryDev{nullptr, nullptr, val.get() + static_cast<uint64_t>(r0 - first) * x.cols, 0, tr, x.cols, x.cols};
    return QueryDev{row_ptr.get() + (r0 - first), col_idx.get(), val.get(), x.row_ptr[first], tr, x.cols, max_row_nnz(x.row_ptr + r0, tr)};
}

// Dense queries are staged tile by tile on the compute stream.  A CSR batch is cut into sub-tiles of `tile` rows or, with
// split (predict), of about a quarter of a batch of >= 4096 rows (at least 1024 rows, at most `tile`), and staged by one of
// three schedules:
//  - whole batch (split, >= 4096 rows, all of them in one tile: predict's common case): the sub-tiles are uploaded on the
//    copy stream into ONE staging set; the UPPER layers (cheap) run per sub-tile as it lands, overlapping the rest of the
//    upload, and the LAST layer -- where the time goes, and where the chunk-major kernel wants as many pairs per launch as
//    it can get -- runs once over the whole batch;
//  - several sub-tiles: they alternate between the two staging sets on the copy stream, the upload of one overlapping the
//    scoring of the previous one;
//  - one sub-tile: one staging set on the compute stream.
void XLinearEngine::for_each_tile_(uint32_t tile, const HostMatrix* x, const TileFn& run, bool split) {
    const size_t all = layers_.size();
    if (!x) {
        for (uint32_t r0 = 0; r0 < resident_.rows; r0 += tile) {
            QueryDev q = resident_;
            q.row_ptr += r0;
            q.rows = std::min(tile, resident_.rows - r0);
            run(Tile{q, r0, 0, 0, all});
        }
        return;
    }
    const uint32_t rows = x->rows, part = ((rows + 3u) / 4u + 31u) & ~31u;
    split = split && !x->dense && rows >= 4096u;
    const bool whole = split && tile >= rows;
    const uint32_t sub = whole ? part : split ? std::min(tile, std::max<uint32_t>(1024u, part)) : tile;
    const bool overlap = !x->dense && rows > sub;
    // room for the largest sub-tile (whole batch: for all of it) before the pipeline starts: a reallocation synchronises
    const uint32_t span = whole ? rows : sub;
    uint64_t n_max = 0;
    for (uint32_t r0 = 0; r0 < rows; r0 += span) {
        const uint32_t tr = std::min(span, rows - r0);
        n_max = std::max(n_max, x->dense ? static_cast<uint64_t>(tr) * x->cols : x->row_ptr[r0 + tr] - x->row_ptr[r0]);
    }
    for (int b = 0; b < (overlap && !whole ? 2 : 1); ++b) stage_[b].reserve(*x, span, n_max);
    uint32_t t = 0;
    for (uint32_t r0 = 0; r0 < rows; r0 += sub, ++t) {
        const uint32_t tr = std::min(sub, rows - r0);
        QueryStage& s = stage_[overlap && !whole ? t & 1u : 0u];
        if (!overlap) {
            run(Tile{s.place(*x, r0, r0, tr, stream_), r0, 0, 0, all});
            continue;
        }
        if (!whole && t >= 2) PB200_CUDA(cudaStreamWaitEvent(copy_stream_, s.consumed, 0));
        const QueryDev q = s.place(*x, whole ? 0 : r0, r0, tr, copy_stream_);
        PB200_CUDA(cudaEventRecord(s.landed, copy_stream_));
        PB200_CUDA(cudaStreamWaitEvent(stream_, s.landed, 0));
        run(whole ? Tile{q, r0, r0, 0, all - 1} : Tile{q, r0, 0, 0, all});
        if (!whole) PB200_CUDA(cudaEventRecord(s.consumed, stream_));
    }
    if (whole) run(Tile{stage_[0].view(*x, 0, 0, rows), 0, 0, all - 1, all});
}

void XLinearEngine::stage_beam_(uint32_t rows, bool with_vals, const BeamFn& fill) {
    PB200_CUDA(cudaStreamSynchronize(stream_));  // the pinned staging area may still feed the previous copy
    const uint64_t n = static_cast<uint64_t>(rows) * beam_stride_;
    beam_id_host_.reserve(n + 1);
    if (with_vals) beam_val_host_.reserve(n + 1);
    beam_cnt_host_.reserve(static_cast<uint64_t>(rows) + 1);
    for (uint32_t r = 0; r < rows; ++r) {
        const uint64_t o = static_cast<uint64_t>(r) * beam_stride_;
        beam_cnt_host_.get()[r] = fill(r, beam_id_host_.get() + o, with_vals ? beam_val_host_.get() + o : nullptr);
    }
    PB200_CUDA(cudaMemcpyAsync(beam_id_[0].get(), beam_id_host_.get(), n * 4, cudaMemcpyHostToDevice, stream_));
    if (with_vals) PB200_CUDA(cudaMemcpyAsync(beam_val_[0].get(), beam_val_host_.get(), n * 4, cudaMemcpyHostToDevice, stream_));
    PB200_CUDA(cudaMemcpyAsync(beam_cnt_[0].get(), beam_cnt_host_.get(), static_cast<uint64_t>(rows) * 4, cudaMemcpyHostToDevice, stream_));
}

XLinearEngine::Result XLinearEngine::predict(const HostMatrix& x, uint32_t beam_size, const char* post_processor, uint32_t only_topk) {
    PB200_CUDA(cudaSetDevice(device_));
    const auto plan = make_plan_(beam_size, post_processor, only_topk);
    const uint32_t rows = x.rows, stride = plan.back().k_cap;
    const OutTarget out = reserve_results_(results_, rows, stride);
    for_each_tile_(ensure_workspace_(plan, rows, x.dense ? x.cols : 0u), &x, [&](const Tile& t) {
        run_tile_(t.q, plan, out.at(t.r0), t.ws_row, false, false, 0, t.d_begin, t.d_end);
    }, /*split=*/true);
    return finish_result_(results_, rows, stride);
}

XLinearEngine::Result XLinearEngine::predict_single_layer(const HostMatrix& x, const HostMatrix& codes, const char* post_processor,
                                                          uint32_t only_topk) {
    PB200_CUDA(cudaSetDevice(device_));
    if (host_->layers.size() != 1) throw std::runtime_error("pecos_b200: predict_single_layer needs a one-layer model");
    const auto& HL = host_->layers[0];
    const uint32_t rows = x.rows;
    const bool have_codes = codes.row_ptr != nullptr;
    // beam entering the layer: the given previous prediction, or every parent with value 1 (libpecos.cpp:209-219)
    uint32_t b_prev = have_codes ? 1u : std::max<uint32_t>(HL.n_chunks, 1u);
    if (have_codes) {
        for (uint32_t r = 0; r < rows; ++r)
            b_prev = std::max<uint32_t>(b_prev, static_cast<uint32_t>(std::min<uint64_t>(codes.row_ptr[r + 1] - codes.row_ptr[r], 0xFFFFFFFFull)));
        const uint64_t n = codes.row_ptr[rows] - codes.row_ptr[0];
        for (uint64_t i = 0; i < n; ++i)
            if (codes.col_idx[codes.row_ptr[0] + i] >= HL.n_chunks)
                throw std::runtime_error("pecos_b200: csr_codes column index >= C.cols");
    }
    // only_topk_to_use = overridden > 0 ? overridden : metadata.only_topk, both = this argument
    const auto plan = make_plan_(0, post_processor, only_topk, {b_prev});
    const uint32_t stride = plan[0].k_cap;
    const OutTarget out = reserve_results_(results_, rows, stride);
    if (only_topk == 0) {  // sorted_csr keeps min(nnz, 0) entries per row (inference.hpp:1237)
        if (rows) PB200_CUDA(cudaMemsetAsync(out.cnt, 0, static_cast<uint64_t>(rows) * 4, stream_));
        return finish_result_(results_, rows, stride);
    }
    for_each_tile_(ensure_workspace_(plan, rows, x.dense ? x.cols : 0u), &x, [&](const Tile& t) {
        const uint32_t r0 = t.r0;
        stage_beam_(t.q.rows, true, [&](uint32_t r, uint32_t* ids, float* vals) {
            if (have_codes) {
                const uint64_t b = codes.row_ptr[r0 + r], e = codes.row_ptr[r0 + r + 1];
                std::memcpy(ids, codes.col_idx + b, (e - b) * 4);
                std::memcpy(vals, codes.val + b, (e - b) * 4);
                return static_cast<uint32_t>(e - b);
            }
            for (uint32_t j = 0; j < HL.n_chunks; ++j) { ids[j] = j; vals[j] = 1.0f; }
            return HL.n_chunks;
        });
        run_tile_(t.q, plan, out.at(r0), 0, false, /*ext_beam=*/true, /*combine_first=*/have_codes ? 1 : 0);
    });
    return finish_result_(results_, rows, stride);
}

void XLinearEngine::resident_upload_csr(const HostMatrix& x) {
    PB200_CUDA(cudaSetDevice(device_));
    has_resident_ = false;
    resident_stage_.reserve(x, x.rows, x.row_ptr[x.rows] - x.row_ptr[0]);
    resident_ = resident_stage_.place(x, 0, 0, x.rows, stream_);
    PB200_CUDA(cudaStreamSynchronize(stream_));
    has_resident_ = true;
}

double XLinearEngine::resident_predict(uint32_t beam_size, const char* post_processor, uint32_t only_topk, bool collect_stats) {
    if (!has_resident_) throw std::runtime_error("pecos_b200: no resident query batch uploaded");
    PB200_CUDA(cudaSetDevice(device_));
    const auto plan = make_plan_(beam_size, post_processor, only_topk);
    resident_stride_ = plan.back().k_cap;
    const OutTarget out = reserve_results_(resident_results_, resident_.rows, resident_stride_);
    const uint32_t tile = ensure_workspace_(plan, resident_.rows, 0);
    if (collect_stats) PB200_CUDA(cudaMemsetAsync(stats_dev_.get(), 0, stats_dev_.bytes(), stream_));
    PB200_CUDA(cudaEventRecord(ev_[3], stream_));
    cudaEvent_t stop;
    PB200_CUDA(cudaEventCreate(&stop));
    for_each_tile_(tile, nullptr, [&](const Tile& t) { run_tile_(t.q, plan, out.at(t.r0), 0, collect_stats); });
    PB200_CUDA(cudaEventRecord(stop, stream_));
    PB200_CUDA(cudaEventSynchronize(stop));
    float ms = 0.f;
    PB200_CUDA(cudaEventElapsedTime(&ms, ev_[3], stop));
    cudaEventDestroy(stop);
    if (collect_stats) {
        std::vector<unsigned long long> h(8 * layers_.size());
        PB200_CUDA(cudaMemcpy(h.data(), stats_dev_.get(), h.size() * 8, cudaMemcpyDeviceToHost));
        for (size_t d = 0; d < layers_.size(); ++d) {
            XLinearStats s{};
            s.chunks = h[8 * d + 0]; s.chunk_rows = h[8 * d + 1]; s.matched = h[8 * d + 2]; s.entries = h[8 * d + 3];
            s.out_cols = h[8 * d + 4]; s.query_nnz = h[8 * d + 5]; s.beam_out = h[8 * d + 6];
            layer_stats_[d] = s;
        }
    }
    return static_cast<double>(ms);
}

uint32_t XLinearEngine::sharded_local_csr_packed(const HostMatrix& x, uint32_t beam_size, const char* post_processor, uint32_t only_topk,
                                                 uint32_t stride_capacity, void* rec_dev) {
    PB200_CUDA(cudaSetDevice(device_));
    const auto plan = make_plan_(beam_size, post_processor, only_topk);
    const uint32_t rows = x.rows, stride = plan.back().k_cap;
    if (stride > stride_capacity) throw std::runtime_error("pecos_b200: sharded output buffers are too narrow for this top-k");
    const uint64_t n = static_cast<uint64_t>(rows) * stride;
    shard_keys_.reserve(n + 1);
    shard_ids_.reserve(n + 1);
    shard_vals_.reserve(n + 1);
    shard_cnt_.reserve(static_cast<uint64_t>(rows) + 1);
    const OutTarget out{shard_ids_.get(), shard_vals_.get(), shard_cnt_.get(), shard_keys_.get(), stride};
    for_each_tile_(ensure_workspace_(plan, rows, 0), &x, [&](const Tile& t) { run_tile_(t.q, plan, out.at(t.r0)); });
    if (n) {
        xl_shard_pack_kernel<<<static_cast<uint32_t>((n + 255) / 256), 256, 0, stream_>>>(
            shard_keys_.get(), shard_ids_.get(), shard_vals_.get(), shard_cnt_.get(), rows, stride, static_cast<ShardRecord*>(rec_dev));
        PB200_CUDA(cudaGetLastError());
        ++launches_;
    }
    PB200_CUDA(cudaStreamSynchronize(stream_));
    return stride;
}

XLinearEngine::Result XLinearEngine::sharded_merge_packed(uint32_t world, uint32_t rows, uint32_t stride, uint32_t only_topk,
                                                          const void* g_rec) {
    PB200_CUDA(cudaSetDevice(device_));
    if (static_cast<uint64_t>(world) * stride > static_cast<uint64_t>(kSelKeys))
        throw std::runtime_error("pecos_b200: world * top-k exceeds the merge kernel's capacity");
    const uint32_t k = only_topk ? only_topk : static_cast<uint32_t>(host_->layers.back().only_topk);
    const uint32_t k_out = std::min<uint32_t>(k, world * stride);
    const OutTarget out = reserve_results_(results_, rows, k_out);
    if (rows) {
        shard_merge_packed_kernel<<<(rows + kSelWarps - 1) / kSelWarps, kSelWarps * 32, 0, stream_>>>(
            static_cast<const ShardRecord*>(g_rec), world, rows, stride, k_out, out.ids, out.vals, out.cnt);
        PB200_CUDA(cudaGetLastError());
        ++launches_;
    }
    return finish_result_(results_, rows, k_out);
}

XLinearEngine::Result XLinearEngine::resident_fetch() {
    PB200_CUDA(cudaSetDevice(device_));
    return finish_result_(resident_results_, resident_.rows, resident_stride_);
}

// predict_on_selected_outputs on the device (SURVEY 8f-2).
//
// Replaces HierarchicalMLModel::predict_on_selected_outputs (pecos/core/xmc/inference.hpp:2507-2571), per layer
// MLModel::predict_on_selected_outputs_internal (:2129-2180) with prolongate_sparse_predictions (:1302-1358); C ABI
// c_xlinear_predict_on_selected_outputs_{csr,drm}_f32 (pecos/core/libpecos.cpp:179-198).
//
// What the reference computes: the scores of exactly the given (query, label) pairs pushed through the hierarchy, no
// top-k.  The selected set of layer l-1 is the SORTED set of parents of layer l's selected set; a row of layer l holds,
// for every entry of the previous layer's row IN ORDER, its children in C's column order that belong to the layer's
// selected set; value = transform(raw score) combined with the parent's value (not at layer 0).
//
// Split used here: everything STRUCTURAL (selected sets, entry order, which candidate position and which parent entry an
// entry reads) depends only on C and the selected pattern, so the host computes it per query; the device does the
// arithmetic with the SAME validated score kernels as beam search -- the previous layer's entry list plays the beam's
// role, so cand[] holds every child of every listed parent in prolongation order -- followed by one small gather kernel
// (xl_selected_gather_kernel: transform + combine of the selected candidates).  Raw scores are therefore bit-identical
// to predict()'s.
XLinearEngine::SelectedResult XLinearEngine::predict_selected(const HostMatrix& x, const HostMatrix& sel, const char* post_processor,
                                                              const HostMatrix& codes) {
    PB200_CUDA(cudaSetDevice(device_));
    // codes (single-layer handles only, c_mlmodel_predict_on_selected_outputs_*): the previous layer's prediction; its
    // rows replace the root as the first layer's parent list and its values are combined with the first layer's scores
    const bool have_codes = codes.row_ptr != nullptr;
    if (have_codes && layers_.size() != 1) throw std::runtime_error("pecos_b200: csr_codes needs a one-layer model");
    const size_t depth = layers_.size();
    const auto& HL = host_->layers;
    const uint32_t rows = x.rows;
    const uint64_t* sel_ptr = sel.row_ptr;
    const uint32_t* sel_idx = sel.col_idx;
    if (sel.cols != HL.back().out_cols) throw std::runtime_error("pecos_b200: selected_outputs_csr.cols != nr_labels");
    if (sel_index_.empty()) {  // label (original numbering of the layer) -> the chunk (= parent node) and column offset that holds it
        sel_index_.resize(depth);
        for (size_t d = 0; d < depth; ++d) {
            const auto& L = HL[d];
            SelIndex& ix = sel_index_[d];
            ix.chunk_of_label.assign(L.out_cols, 0xFFFFFFFFu);  // 0xFFFFFFFF: the label has no parent (pruned tree)
            ix.offset_of_label.assign(L.out_cols, 0u);
            for (uint32_t p = 0; p < L.n_chunks; ++p) {
                const ChunkHeader& h = L.chunks[p];
                for (uint32_t j = 0; j < h.n_cols; ++j) {
                    const uint32_t col = h.col_begin + j;
                    const uint32_t label = L.reordered ? L.label_of_col[col] : col;
                    if (label < L.out_cols) { ix.chunk_of_label[label] = p; ix.offset_of_label[label] = j; }
                }
            }
        }
    }
    SelectedResult out;
    out.rows = rows;
    out.cols = sel.cols;
    out.indptr.assign(sel_ptr, sel_ptr + rows + 1);
    const uint64_t sel_base = sel_ptr[0];
    for (auto& v : out.indptr) v -= sel_base;
    const uint64_t total = out.indptr[rows];
    out.indices.assign(total, 0u);
    out.data.assign(total, 0.0f);
    if (rows == 0) return out;

    // ---- structure, per query (host threads): entry lists of every layer
    struct Lists {
        std::vector<uint64_t> ptr;       // [rows + 1]
        std::vector<uint32_t> id;        // label of the entry (original numbering of the layer)
        std::vector<uint32_t> pos;       // candidate position inside the query's row of this layer
        std::vector<uint32_t> parent;    // index of the parent entry inside the query's row of the previous layer
    };
    std::vector<Lists> lists(depth);
    {
        std::vector<std::vector<uint32_t>> q_id(static_cast<size_t>(rows) * depth), q_pos(static_cast<size_t>(rows) * depth),
            q_par(static_cast<size_t>(rows) * depth);
        const unsigned hw = std::max(1u, std::min(32u, std::thread::hardware_concurrency()));
        const unsigned n_thr = static_cast<unsigned>(std::min<uint64_t>(hw, std::max<uint64_t>(1, rows / 64)));
        std::vector<std::thread> pool;
        std::atomic<uint32_t> next{0};
        std::vector<std::exception_ptr> errs(n_thr);
        auto work = [&](unsigned t) {
            try {
                std::vector<std::vector<uint32_t>> sel(depth);
                for (;;) {
                    const uint32_t q0 = next.fetch_add(64);
                    if (q0 >= rows) break;
                    for (uint32_t q = q0; q < std::min(rows, q0 + 64); ++q) {
                        // selected sets, leaf upwards (sorted, unique)
                        sel[depth - 1].assign(sel_idx + sel_ptr[q], sel_idx + sel_ptr[q + 1]);
                        for (uint32_t lab : sel[depth - 1])
                            if (lab >= HL.back().out_cols) throw std::runtime_error("pecos_b200: selected label id out of range");
                        std::sort(sel[depth - 1].begin(), sel[depth - 1].end());
                        for (size_t d = depth - 1; d > 0; --d) {
                            auto& up = sel[d - 1];
                            up.clear();
                            for (uint32_t lab : sel[d]) {
                                const uint32_t par = sel_index_[d].chunk_of_label[lab];
                                if (par != 0xFFFFFFFFu) up.push_back(par);
                            }
                            std::sort(up.begin(), up.end());
                            up.erase(std::unique(up.begin(), up.end()), up.end());
                        }
                        // entry lists, root downwards; first parent list: the given codes row, else every code of the first
                        // layer (= the root for a hierarchical model; ones(rows x nr_codes) for a single layer, libpecos.cpp:96-99)
                        std::vector<uint32_t> prev_id;
                        if (have_codes) prev_id.assign(codes.col_idx + codes.row_ptr[q], codes.col_idx + codes.row_ptr[q + 1]);
                        else { prev_id.resize(HL[0].n_chunks); for (uint32_t p = 0; p < HL[0].n_chunks; ++p) prev_id[p] = p; }
                        for (size_t d = 0; d < depth; ++d) {
                            auto& ids = q_id[static_cast<size_t>(q) * depth + d];
                            auto& pos = q_pos[static_cast<size_t>(q) * depth + d];
                            auto& par = q_par[static_cast<size_t>(q) * depth + d];
                            const auto& L = HL[d];
                            const auto& S = sel[d];
                            uint32_t slot_base = 0;
                            for (uint32_t i = 0; i < prev_id.size(); ++i) {
                                const uint32_t p = prev_id[i];
                                if (p >= L.n_chunks) throw std::runtime_error("pecos_b200: selected outputs: parent id out of range");
                                const ChunkHeader& h = L.chunks[p];
                                for (uint32_t j = 0; j < h.n_cols; ++j) {
                                    const uint32_t col = h.col_begin + j;
                                    const uint32_t label = L.reordered ? L.label_of_col[col] : col;
                                    if (ids.size() >= S.size() || !std::binary_search(S.begin(), S.end(), label)) continue;
                                    ids.push_back(label);
                                    pos.push_back(slot_base + j);
                                    par.push_back(i);
                                }
                                slot_base += h.n_cols;
                            }
                            prev_id = ids;
                        }
                    }
                }
            } catch (...) { errs[t] = std::current_exception(); }
        };
        for (unsigned t = 1; t < n_thr; ++t) pool.emplace_back(work, t);
        work(0);
        for (auto& th : pool) th.join();
        for (auto& e : errs) if (e) std::rethrow_exception(e);
        for (size_t d = 0; d < depth; ++d) {
            auto& Ls = lists[d];
            Ls.ptr.assign(static_cast<size_t>(rows) + 1, 0);
            for (uint32_t q = 0; q < rows; ++q) Ls.ptr[q + 1] = Ls.ptr[q] + q_id[static_cast<size_t>(q) * depth + d].size();
            Ls.id.resize(Ls.ptr[rows]);
            Ls.pos.resize(Ls.ptr[rows]);
            Ls.parent.resize(Ls.ptr[rows]);
            for (uint32_t q = 0; q < rows; ++q) {
                const size_t k = static_cast<size_t>(q) * depth + d;
                std::copy(q_id[k].begin(), q_id[k].end(), Ls.id.begin() + Ls.ptr[q]);
                std::copy(q_pos[k].begin(), q_pos[k].end(), Ls.pos.begin() + Ls.ptr[q]);
                std::copy(q_par[k].begin(), q_par[k].end(), Ls.parent.begin() + Ls.ptr[q]);
            }
        }
    }

    // ---- plan: the beam entering layer d is the entry list of layer d - 1 (layer 0: the codes rows, else every parent)
    std::vector<uint32_t> b_in(depth, 1u);
    for (size_t d = 0; d < depth; ++d) {
        uint32_t& b = b_in[d];
        if (d > 0)
            for (uint32_t q = 0; q < rows; ++q) b = std::max<uint32_t>(b, static_cast<uint32_t>(lists[d - 1].ptr[q + 1] - lists[d - 1].ptr[q]));
        else if (have_codes)
            for (uint32_t q = 0; q < rows; ++q) b = std::max<uint32_t>(b, static_cast<uint32_t>(codes.row_ptr[q + 1] - codes.row_ptr[q]));
        else
            b = std::max<uint32_t>(1u, HL[0].n_chunks);
    }
    const auto plan = make_plan_(1, post_processor, 1, b_in, /*topk=*/false);

    DeviceBuffer<uint64_t> d_ptr[2];
    DeviceBuffer<uint32_t> d_pos, d_par;
    DeviceBuffer<float> d_val[2];
    std::vector<uint64_t> rel_ptr;
    std::vector<float> leaf_vals;
    for_each_tile_(ensure_workspace_(plan, rows, x.dense ? x.cols : 0u), &x, [&](const Tile& t) {
        const QueryDev& qd = t.q;
        const uint32_t r0 = t.r0, tr = qd.rows;
        int cur = 0;  // which d_ptr / d_val set holds the previous layer
        if (have_codes) {  // the given previous prediction plays "layer -1"
            const uint64_t c0 = codes.row_ptr[r0], c1 = codes.row_ptr[r0 + tr];
            rel_ptr.resize(static_cast<size_t>(tr) + 1);
            for (uint32_t r = 0; r <= tr; ++r) rel_ptr[r] = codes.row_ptr[r0 + r] - c0;
            d_ptr[cur].upload(rel_ptr.data(), rel_ptr.size(), stream_);
            d_val[cur].upload(codes.val + c0, c1 - c0, stream_);
        }
        for (size_t d = 0; d < depth; ++d) {
            // beam = the previous layer's entry list (layer 0: the codes rows, else every parent); also waits for the
            // previous layer, whose uploads came from rel_ptr
            stage_beam_(tr, false, [&](uint32_t r, uint32_t* ids, float*) {
                const uint64_t* ptr = d > 0 ? lists[d - 1].ptr.data() : have_codes ? codes.row_ptr : nullptr;
                if (!ptr) {
                    for (uint32_t p = 0; p < HL[0].n_chunks; ++p) ids[p] = p;
                    return HL[0].n_chunks;
                }
                const uint64_t b = ptr[r0 + r], n = ptr[r0 + r + 1] - b;
                std::memcpy(ids, (d > 0 ? lists[d - 1].id.data() : codes.col_idx) + b, n * 4);
                return static_cast<uint32_t>(n);
            });
            const TileShape one_layer{/*ext_beam=*/true, 0, d, d + 1, false, /*topk=*/false};
            score_layer_(d, qd, plan, pick_kernels_(d, qd, plan, one_layer), 0, 0, false);
            const auto& Ls = lists[d];
            const uint64_t e0 = Ls.ptr[r0], e1 = Ls.ptr[r0 + tr];
            rel_ptr.resize(static_cast<size_t>(tr) + 1);
            for (uint32_t r = 0; r <= tr; ++r) rel_ptr[r] = Ls.ptr[r0 + r] - e0;
            const int nxt = cur ^ 1;
            d_ptr[nxt].upload(rel_ptr.data(), rel_ptr.size(), stream_);
            d_pos.upload(Ls.pos.data() + e0, e1 - e0, stream_);
            d_par.upload(Ls.parent.data() + e0, e1 - e0, stream_);
            d_val[nxt].reserve(std::max<uint64_t>(e1 - e0, 1));
            const uint64_t cand_stride_q = static_cast<uint64_t>(plan[d].b_prev) * std::max<uint32_t>(layers_[d].view.c_max, 1u);
            xl_selected_gather_kernel<<<tr, 128, 0, stream_>>>(cand_.get(), cand_stride_q, d_ptr[nxt].get(), d_pos.get(), d_par.get(),
                                                             d_ptr[cur].get(), d_val[cur].get(), d_val[nxt].get(), plan[d].pp.kind,
                                                             plan[d].pp.p, (d > 0 || have_codes) ? 1 : 0);
            PB200_CUDA(cudaGetLastError());
            ++launches_;
            cur = nxt;
        }
        // leaf values of this tile -> result rows (the reference copies the selected row's LENGTH; entries it could not reach
        // -- labels without a path to the root -- stay zero, inference.hpp:2560-2568)
        const auto& Lf = lists[depth - 1];
        const uint64_t e0 = Lf.ptr[r0], e1 = Lf.ptr[r0 + tr];
        leaf_vals.resize(e1 - e0);
        PB200_CUDA(cudaStreamSynchronize(stream_));
        if (e1 > e0) PB200_CUDA(cudaMemcpy(leaf_vals.data(), d_val[cur].get(), (e1 - e0) * 4, cudaMemcpyDeviceToHost));
        for (uint32_t r = 0; r < tr; ++r) {
            const uint64_t ob = out.indptr[r0 + r], on = out.indptr[r0 + r + 1] - ob;
            const uint64_t lb = Lf.ptr[r0 + r], ln = Lf.ptr[r0 + r + 1] - lb;
            for (uint64_t i = 0; i < std::min(on, ln); ++i) {
                out.indices[ob + i] = Lf.id[lb + i];
                out.data[ob + i] = leaf_vals[lb - e0 + i];
            }
        }
    });
    return out;
}

}  // namespace pb200

#ifdef PB200_CM_TRACE
// diagnostics build only (tools/profile_cm_kernel.py): copies the chunk-major score kernel's trace (see CmTrace) to out
extern "C" int pb200_cm_trace_fetch(unsigned long long* out, unsigned long long n) {
    const unsigned long long cap = sizeof(pb200::g_cm_trace) / sizeof(unsigned long long);
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    return cudaMemcpyFromSymbol(out, pb200::g_cm_trace, (n < cap ? n : cap) * sizeof(unsigned long long)) == cudaSuccess ? 0 : -1;
}
#endif
