// xl_query_warp_scores_kernel: one WARP walks one query through ALL the chunks of its beam at once.
//
// Included by xlinear_engine.cu (inside its anonymous namespace, after the small device helpers).
//
// Why: scoring a (query, chunk) pair of a narrow chunk touches a few dozen {col, val} entries, and the per-pair
// bookkeeping of the warp-per-chunk kernel (flush set-up, scans) costs more than the arithmetic.  Here one warp probes
// the chunks of the beam one after the other -- lane = query feature, one 8-byte feature-map cell per probe, the probes of
// two chunks (8 loads per lane) in flight together -- and collects the matches of SEVERAL chunks before it applies them:
//
//   * lanes of one load instruction probe the SAME chunk with ascending features, so the popular (small) feature ids
//     share 128-byte lines: the L1 pipeline, which processes one line per ~2 cycles and instruction, sees about half the
//     lines of a lane-per-chunk arrangement (measured limiter: 2,560 probes per query and layer);
//   * matches are chunk-major, feature-ascending inside a chunk; entries of different chunks hit different columns, and
//     entries of one 32-group that hit the same column are added in concatenation order (__match_any_sync), i.e. in
//     ascending feature order;
//   * the apply pass is entry-parallel (lane = entry of the concatenated matched rows, row found by a binary search in
//     the prefix sums), so ragged rows cost the same per entry and nothing is staged.
//
// Arithmetic order per output column is unchanged: matched features ascending, un-fused multiply and add, bias row last
// (pecos/core/xmc/inference.hpp:788-811).  Eligibility (checked on the host, otherwise the warp-per-chunk kernel runs):
// sparse queries, feature maps present, beam <= kQwSlots, candidate row <= kQwNCap floats, query nnz <= kQwQCap.
#pragma once

constexpr int kQwWarps = 4;        // queries per CTA
constexpr int kQwSlots = 32;       // beam slots (one lane per slot)
constexpr int kQwPairs = 128;      // matched rows collected per apply pass
constexpr uint32_t kQwNCap = 2048; // candidate row capacity (floats)
constexpr uint32_t kQwQCap = 512;  // query non-zeros staged per warp

struct QwSlot {
    const uint2* fm;       // feature-map cells of the chunk (nullptr: nothing to probe)
    const uint2* ext;      // {first entry, end} of every chunk row, relative to ent
    const uint2* ent;      // entries of the chunk
    uint32_t base;         // first candidate position of this slot
    uint32_t n_rows;       // R
};

__host__ __device__ inline size_t qw_warp_bytes(uint32_t q_cap, uint32_t n_cap) {
    return static_cast<size_t>(q_cap) * 8                      // qidx + qval
           + sizeof(QwSlot) * kQwSlots                          // slots
           + static_cast<size_t>(kQwPairs) * 8                  // {row, slot} of a match; becomes the row's entry pointer
           + static_cast<size_t>(kQwPairs) * (4 + 4)            // mx, mb
           + static_cast<size_t>(kQwPairs + 4) * 4              // off
           + static_cast<size_t>(n_cap) * 4;                    // out
}

template <bool STATS>
__global__ void __launch_bounds__(kQwWarps * 32, 8)  // <= 64 registers, ~5 KB of shared memory per warp => 32 warps per SM
xl_query_warp_scores_kernel(const LayerDev L, const QueryDev X, const uint32_t* __restrict__ beam_id,
                            const uint32_t* __restrict__ beam_cnt, const uint32_t beam_stride, float* __restrict__ cand,
                            const uint64_t cand_stride_q, unsigned long long* stats, const uint32_t q_cap,
                            const uint32_t n_cap, const uint32_t rows) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const uint32_t q = blockIdx.x * kQwWarps + warp;
    if (q >= rows) return;
    const size_t slice = (qw_warp_bytes(q_cap, n_cap) + 15) & ~static_cast<size_t>(15);
    unsigned char* base_ptr = smem_raw + warp * slice;
    uint32_t* qidx = reinterpret_cast<uint32_t*>(base_ptr);
    float* qval = reinterpret_cast<float*>(qidx + q_cap);
    QwSlot* slots = reinterpret_cast<QwSlot*>(qval + q_cap);
    uint2* mrow = reinterpret_cast<uint2*>(slots + kQwSlots);            // {chunk row, beam slot} of a match ...
    const uint2** ment = reinterpret_cast<const uint2**>(mrow);          // ... overwritten by the row's first entry
    float* mx = reinterpret_cast<float*>(mrow + kQwPairs);               // multiplier
    uint32_t* mb = reinterpret_cast<uint32_t*>(mx + kQwPairs);           // first candidate position of the match's slot
    uint32_t* off = mb + kQwPairs;                                       // entry prefix
    float* out = reinterpret_cast<float*>(off + kQwPairs + 4);           // candidate row of this query

    // ---- prologue: all global loads first, shared-memory stores afterwards (issue is in order)
    const uint32_t cnt = min(beam_cnt[q], static_cast<uint32_t>(kQwSlots));
    const uint64_t qb = X.row_ptr[q] - X.nnz_base;
    const int qn = static_cast<int>(X.row_ptr[q + 1] - X.nnz_base - qb);
    const uint32_t my_p = (static_cast<uint32_t>(lane) < cnt) ? beam_id[static_cast<uint64_t>(q) * beam_stride + lane] : 0u;
    ChunkHeader my_h;
    my_h.n_cols = 0; my_h.nnz_rows = 0; my_h.has_bias = 0; my_h.meta_off = 0; my_h.ent_off = 0; my_h.col_begin = 0;
    if (static_cast<uint32_t>(lane) < cnt) my_h = L.chunks[my_p];
    for (int i0 = lane; i0 < qn; i0 += 128) {
        uint32_t fi[4];
        float fv[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) { const int i = i0 + 32 * u; fi[u] = (i < qn) ? X.col_idx[qb + i] : 0u; fv[u] = (i < qn) ? X.val[qb + i] : 0.0f; }
#pragma unroll
        for (int u = 0; u < 4; ++u) { const int i = i0 + 32 * u; if (i < qn) { qidx[i] = fi[u]; qval[i] = fv[u]; } }
    }
    // slot table + exclusive prefix of the chunk widths (candidate positions are global over the beam)
    const uint32_t incl = warp_incl_scan(my_h.n_cols, lane);
    const uint32_t n_total = __shfl_sync(kFull, incl, 31);
    const bool scored = static_cast<uint32_t>(lane) < cnt && !(my_h.has_bias & kChunkAbsent);  // absent: another GPU's chunk
    const bool probing = scored && my_h.nnz_rows > 0;
    if (static_cast<uint32_t>(lane) < cnt) {
        QwSlot s;
        s.fm = probing ? L.featmap + static_cast<uint64_t>(my_p) * L.fm_words : nullptr;
        s.ext = reinterpret_cast<const uint2*>(L.rowext + my_h.meta_off);
        s.ent = L.entries + my_h.ent_off;
        s.base = incl - my_h.n_cols;
        s.n_rows = my_h.nnz_rows;
        slots[lane] = s;
    }
    for (uint32_t i = lane; i < n_total; i += 32) out[i] = 0.0f;
    __syncwarp();

    unsigned long long st_match = 0, st_ent = 0;

    // Applies the m matches collected in (mrow, mx), which are in feature-major order.
    auto flush = [&](int m) {
        if (m == 0) return;
        __syncwarp();
        // row extents (4 matches per lane, all loads in flight), prefix over the matches
        constexpr int PER = kQwPairs / 32;
        const uint2* a[PER];
        uint32_t c[PER], bs[PER];
        uint32_t local = 0;
#pragma unroll
        for (int u = 0; u < PER; ++u) {
            const int i = lane * PER + u;
            a[u] = nullptr; c[u] = 0; bs[u] = 0;
            if (i < m) {
                const uint2 rj = mrow[i];
                const QwSlot sl = slots[rj.y];
                const uint2 lh = __ldg(sl.ext + rj.x);  // one 8-byte load per matched row
                a[u] = sl.ent + lh.x; c[u] = lh.y - lh.x; bs[u] = sl.base;
            }
            local += c[u];
        }
        const uint32_t inc = warp_incl_scan(local, lane);
        uint32_t run = inc - local;
        const uint32_t total = __shfl_sync(kFull, inc, 31);
        __syncwarp();
#pragma unroll
        for (int u = 0; u < PER; ++u) {
            const int i = lane * PER + u;
            if (i < m) { ment[i] = a[u]; mb[i] = bs[u]; off[i] = run; run += c[u]; }
        }
        if (lane == 0) off[m] = total;
        __syncwarp();
        st_ent += total;
        st_match += m;

        for (uint32_t g0 = 0; g0 < total; g0 += 128u) {
            uint2 e[4];
            float x[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {  // four independent (search, load) chains in flight per lane
                const uint32_t g = g0 + 32u * u + lane;
                e[u] = make_uint2(0xFFFFFFFFu - lane, 0u);  // idle lanes: distinct pseudo-targets, never applied
                x[u] = 0.0f;
                if (g < total) {
                    // independent binary searches: this kernel is latency-bound (32 warps/SM), and the serial row-start
                    // mask chain of xl_rows_of_group slower here (S layers 2-4)
                    const int i = last_le_u32(off, m, g);  // off[i] <= g < off[i + 1]
                    e[u] = __ldg(ment[i] + (g - off[i]));
                    e[u].x += mb[i];
                    x[u] = mx[i];
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
        __syncwarp();
    };

    // ---- probes: two chunks per step, lane = query feature (4 x 32 features per chunk and pass)
    if (__ballot_sync(kFull, probing) != 0u && qn > 0) {
        int m = 0;
        for (uint32_t j0 = 0; j0 < cnt; j0 += 2) {
            const uint2* fm[2];
            fm[0] = slots[j0].fm;
            fm[1] = (j0 + 1 < cnt) ? slots[j0 + 1].fm : nullptr;
            if (fm[0] == nullptr && fm[1] == nullptr) continue;
            for (int tb = 0; tb < qn; tb += 128) {
                uint32_t bitpos[4];
                uint32_t word[4];
                bool live[4];
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const int t = tb + 32 * u + lane;
                    live[u] = false; bitpos[u] = 0; word[u] = 0;
                    if (t < qn) {
                        const uint32_t f = qidx[t];
                        const bool dup = (t > 0) && (qidx[t - 1] == f);  // only the first of repeated indices counts
                        live[u] = !dup && f < L.w_rows;
                        bitpos[u] = f & 31u;
                        word[u] = f >> 5;
                    }
                }
                uint2 cell[2][4];
#pragma unroll
                for (int c = 0; c < 2; ++c) {
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        cell[c][u] = make_uint2(0u, 0u);
                        if (fm[c] != nullptr && live[u]) cell[c][u] = __ldg(fm[c] + word[u]);
                    }
                }
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    if (fm[c] == nullptr) continue;
#pragma unroll
                    for (int u = 0; u < 4; ++u) {
                        if (tb + 32 * u >= qn) break;
                        const bool hit = (cell[c][u].x >> bitpos[u]) & 1u;
                        const unsigned mask = __ballot_sync(kFull, hit);
                        if (mask == 0u) continue;
                        if (hit) {
                            const uint32_t pos = m + __popc(mask & ((1u << lane) - 1u));
                            mrow[pos] = make_uint2(cell[c][u].y + __popc(cell[c][u].x & ((1u << bitpos[u]) - 1u)), j0 + c);
                            mx[pos] = qval[tb + 32 * u + lane];
                        }
                        m += __popc(mask);
                        if (m > kQwPairs - 32) { flush(m); m = 0; }
                    }
                }
            }
        }
        flush(m);
    }
    // ---- bias rows last: one pseudo-feature for every chunk with an explicit bias row
    {
        const bool has = scored && (my_h.has_bias & 1u);
        const unsigned mask = __ballot_sync(kFull, has);
        if (mask) {
            __syncwarp();
            if (has) {
                const uint32_t pos = __popc(mask & ((1u << lane) - 1u));
                mrow[pos] = make_uint2(my_h.nnz_rows - 1u, static_cast<uint32_t>(lane));
                mx[pos] = L.bias;
            }
            flush(__popc(mask));
        }
    }
    __syncwarp();
    float* dst = cand + static_cast<uint64_t>(q) * cand_stride_q;
    for (uint32_t i = lane; i < n_total; i += 32) dst[i] = out[i];
    if (STATS) {
        // per-query counters of SURVEY 8(d); absent chunks (index sharding) are not scored and not counted
        unsigned long long rows_sum = 0, cols_sum = 0, chunks = 0;
        if (scored) { rows_sum = my_h.nnz_rows; cols_sum = my_h.n_cols; chunks = 1; }
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) {
            rows_sum += __shfl_xor_sync(kFull, rows_sum, d);
            cols_sum += __shfl_xor_sync(kFull, cols_sum, d);
            chunks += __shfl_xor_sync(kFull, chunks, d);
        }
        if (lane == 0) {
            atomicAdd(&stats[0], chunks);
            atomicAdd(&stats[1], rows_sum);
            atomicAdd(&stats[2], st_match);
            atomicAdd(&stats[3], st_ent);
            atomicAdd(&stats[4], cols_sum);
            if (cnt > 0) atomicAdd(&stats[5], static_cast<unsigned long long>(qn));
        }
    }
}
