// Chunk-major scoring: the (query, beam slot) pairs of a layer are bucketed by weight chunk, a CTA stages ONE chunk in
// shared memory and every LANE walks ITS OWN pair.
//
// Included by xlinear_engine.cu (inside its anonymous namespace, after the small device helpers).
//
// Why: the query-major kernels spend 600 - 3,900 warp-instructions per pair on match compaction, prefix
// sums and on putting colliding entries of a 32-entry group back into feature order, and every probe / extent / entry
// access is a scattered global load (one L1 line each).  Here
//   * at LOAD time every chunk of an eligible layer is packed into a self-contained IMAGE in HBM (xl_cm_build_images_kernel):
//     header | lookup structure | entry weights (f32) | entry columns (u8).  Lookup structure: for feature spaces up to
//     kCmDirectRows a direct table of w_rows + 1 u16 row starts, feature f's entries = [T[f], T[f + 1]) (a feature without a
//     row gets the next row's start: an empty range); else the chunk's feature map (one bit per feature + a 16-bit row
//     prefix per 32 features: "is f a row, and which one" = one shared-memory word + popcount) and 16-bit row pointers;
//   * per call the pairs are bucketed by chunk on the device (count -> scan -> scatter; the reference's b_sort_by_chunk,
//     pecos/core/xmc/inference.hpp:985-993);
//   * the score kernel is PERSISTENT: one CTA per SM starts on the chunk where its 1/grid share of the estimated work
//     begins (a pair's cost grows with its chunk's entry count: cm_pair_cost), stages that chunk's image by ONE bulk
//     asynchronous copy (cp.async.bulk + mbarrier, the TMA engine's non-tensor form), and its warps CLAIM 32-pair slices of
//     the chunk from a per-chunk cursor (one atomicAdd per slice) until the chunk runs dry; then the CTA moves to the chunk
//     with the most unclaimed estimated work per CTA on it (a per-chunk count of the CTAs there).  Work moves between SMs at
//     run time, so the launch ends when the last slice does, not when the CTA with the most expensive static share does;
//   * a lane walks its pair's query features in ascending order (staged global -> shared by cp.async, rounds of 8 in
//     flight), compacts the hits of a round in place as {entry range, x}, then streams the hit rows' entries as one flat
//     stream, kCmSlots entries per trip across row boundaries AND across rounds: after round r's lookup the warp runs only
//     the trips that finish round r - 1's hits, a lane done early going on into round r's, so the trip count follows the
//     largest backlog of a lane rather than each round's busiest lane; one drain (with the bias row) ends the pair.  The
//     entries go into the lane's PRIVATE accumulators acc[column][lane].  That is the reference's marching loop
//     (inference.hpp:788-811): ascending feature order, separate multiply and add, bias row last; a column is only ever
//     touched by the lane that owns the pair: no compaction across lanes, no conflict resolution.  The scores leave through
//     a shared-memory tile, 8 consecutive columns of 4 pairs per store instruction.
//
// Bit-identical to the query-major kernels (tests/test_chunk_major_gpu.py).  Eligibility: shape (cm_shape, at load: width
// <= 256, rows / entries per chunk < 65535, image + 4 warps fit in shared memory, images within PB200_CMIMG_MB) and call
// (cm_plan: sparse queries, enough pairs per chunk and per SM).
#pragma once

constexpr int kCmFeat = 8;                  // query features staged per pair and round (two rounds in flight per warp)
constexpr int kCmSlots = 4;                 // entries a lane adds per iteration of the accumulate phase
constexpr int kCmMaxWarps = 16;
constexpr int kCmMinWarps = 4;
constexpr uint32_t kCmMaxDup = 400;         // a column cap may at most quadruple the (virtual) chunks of a layer
constexpr uint32_t kCmSmemBudget = 224u << 10;  // dynamic shared memory a CTA may take (227 KB is the sm_90a maximum)
constexpr uint32_t kCmMinReuse = 24;        // average pairs per chunk below which the per-chunk staging does not pay
constexpr uint32_t kCmMinPairsPerSm = 48u;  // fewer pairs than this per SM: the query-major kernels fill the GPU better
constexpr uint32_t kCmDirectRows = 16384;   // feature spaces up to this size get a direct feature -> entry-range table
constexpr uint32_t kCmEmpty = 0xFFFFFFFFu;

struct CmWork {
    uint32_t* slot_pos;     // [rows x beam_stride] first candidate position of every beam slot
    uint32_t* count;        // [n_chunks] pairs per chunk, reused as the scatter cursor
    uint32_t* bucket_ptr;   // [n_chunks + 1]
    uint64_t* cost_ptr;     // [n_chunks + 1] exclusive prefix of the chunks' estimated work (cm_pair_cost x pairs)
    uint32_t* pair_q;       // [pairs] query of a pair, grouped by chunk
    uint32_t* pair_pos;     // [pairs] candidate position of the pair's first column inside the query's row
    uint32_t* claim;        // [n_chunks] first unclaimed pair of a chunk's bucket (at or past bucket_ptr[c + 1]: none left)
    uint32_t* active;       // [n_chunks] CTAs of the score kernel currently on the chunk
};

struct CmPlan {  // per call
    bool eligible = false;
    uint32_t warps = 0, grid = 0;
    size_t smem = 0;
};

// PREFIX mode of xl_cm_scores_kernel: the image is the merged one-chunk layer of layers 0 and 1 (layer 0's n0 columns, then
// layer 1's columns in layer-1 column order, see build_prefix_layer) and pair i is query i of the tile.  A query's layer-0
// beam holds all n0 candidates, so layer 0's top-k is a sort of its n0 transformed scores, and layer 1's beam slots are every
// layer-1 chunk in that order.  The epilogue writes the layer-0 beam and layer 1's raw scores at the candidate positions
// layer 1's top-k kernel reads.
constexpr uint32_t kCmPrefixTop0 = 8;       // widest layer 0 the prefix takes (its keys are sorted in registers)
struct CmPrefixOut {
    uint32_t rows = 0;                      // queries of the tile
    uint32_t n0 = 0;                        // layer 0's columns (<= kCmPrefixTop0)
    int pp_kind = 0, pp_p = 0;              // layer 0's post-processor
    const ChunkHeader* chunks1 = nullptr;   // layer 1's chunks: chunk j = the children of layer-0 column j
    uint32_t* beam_id = nullptr;            // layer 0's beam [rows x beam_stride], best first
    float* beam_val = nullptr;
    uint32_t* beam_cnt = nullptr;
    uint32_t beam_stride = 0;
    float* cand1 = nullptr;                 // layer 1's candidate rows [rows x cand1_stride]
    uint64_t cand1_stride = 0;
};

__host__ __device__ inline uint32_t cm_align16(uint32_t x) { return (x + 15u) & ~15u; }

// staging buffers of a warp: `stages` rounds of query features in flight or in lookup, plus one that still holds the
// previous round's compacted hits (carried into the next round's accumulate trips)
__host__ __device__ constexpr uint32_t cm_buffers(uint32_t stages) { return stages + 1u; }

__host__ __device__ inline size_t cm_warp_bytes(uint32_t acc_cols, uint32_t stages) {
    return static_cast<size_t>(cm_buffers(stages)) * 32 * (kCmFeat + 1) * 8  // staging ring: query features / compacted hits, stride 9
           + static_cast<size_t>(acc_cols) * 32 * 4;                        // accumulators [col][lane]
}

// col_cap: a chunk wider than col_cap columns is cut into ceil(n_cols / col_cap) column ranges of (nearly) equal width, each
// with its OWN image (only its entries) -- a "virtual chunk"; a (query, chunk) pair is then scored once per range.  The lookups
// are repeated for the cut chunks, the accumulate work is not, and both the image and the per-warp accumulators shrink to the
// cap, so more warps fit.  The load path takes the largest cap that fits (cm_layer_layout): a layer is only cut when its
// widest chunk does not fit next to kCmMinWarps warps.  e_max = most entries of one virtual chunk, n_vc = number of virtual
// chunks.
inline CmShape cm_shape(uint32_t fm_words, uint32_t w_rows, uint32_t r_max, uint32_t e_max, uint32_t col_cap, uint32_t n_chunks,
                        uint32_t n_vc) {
    CmShape s;
    if (fm_words == 0 || n_chunks == 0 || col_cap == 0 || col_cap > 256u || r_max >= 65535u || e_max >= 65535u) return s;
    s.direct = w_rows <= kCmDirectRows;
    s.words = s.direct ? w_rows + 1u : fm_words;
    s.col_cap = col_cap;
    s.n_vc = n_vc;
    s.r_cap = r_max; s.e_cap = e_max; s.acc_cols = col_cap;
    // narrow chunks do little arithmetic per round of query features: keep four rounds of cp.async in flight per warp to
    // cover the global-memory latency; wide chunks (long accumulate phases) get by with two
    s.stages = s.acc_cols <= 16u ? 4u : 2u;
    uint32_t off = 16;  // header {bias range, n_cols, R, E}
    s.off_lookup = off; off += cm_align16(s.words * (s.direct ? 2u : 4u));
    if (!s.direct) {
        s.off_pre = off; off += cm_align16(s.words * 2u);
        s.off_rp = off;  off += cm_align16((r_max + 2u) * 2u);
    }
    s.off_ew = off; off += cm_align16((e_max + 1u) * 4u);
    s.off_ec = off; off += cm_align16(e_max + 1u);
    s.img_bytes = (off + 127u) & ~127u;
    if (s.img_bytes + kCmMinWarps * cm_warp_bytes(s.acc_cols, s.stages) + 64 > kCmSmemBudget) return s;
    s.warps_fit = static_cast<uint32_t>(std::min<size_t>(kCmMaxWarps, (kCmSmemBudget - s.img_bytes - 64) / cm_warp_bytes(s.acc_cols, s.stages)));
    s.ok = true;
    return s;
}

// The chunk images a layer with a feature map gets at load time: their shape (vc_ptr unset; ok == false: none fits) and the
// host table of the first virtual chunk of every chunk, [n_chunks + 1] (empty when !shape.ok).
struct CmLayout { CmShape shape; std::vector<uint32_t> vc_ptr; };

// Policy: the LARGEST column cap that fits at all (no cut whenever the layer fits uncut), down in steps of 7/8 until the
// cut would more than quadruple the layer's chunks (kCmMaxDup) or the cap drops below 8.  Cutting gives more warps per CTA,
// but every cut repeats the pair's lookups.  Measured on an H100 80GB HBM3 at 400 W (eurlex-4k leaf, chunks of 46 - 84
// columns, work-weighted CTA shares): uncut, 6 warps, 0.82 ms; cap 42, 15 warps, 1.08 ms; cap 28, 16 warps, 1.07 ms -- the
// kernel is bound by the shared-memory accesses of lookups and entries, not by its warps.
inline CmLayout cm_layer_layout(const ChunkedLayerHost& L) {
    // virtual chunks under column cap `cap`; on request the vc_ptr table and the most entries of one column range
    auto layout_for_cap = [&L](uint32_t cap, std::vector<uint32_t>* vc_ptr_out, uint32_t* e_max_out) {
        uint32_t n_vc = 0, best = 0;
        std::vector<uint32_t> cnt;
        if (vc_ptr_out) vc_ptr_out->assign(static_cast<size_t>(L.n_chunks) + 1, 0u);
        for (uint32_t p = 0; p < L.n_chunks; ++p) {
            const ChunkHeader& ch = L.chunks[p];
            if (vc_ptr_out) (*vc_ptr_out)[p] = n_vc;
            if ((ch.has_bias & kChunkAbsent) || ch.n_cols == 0) continue;
            const uint32_t nr = (ch.n_cols + cap - 1) / cap;
            n_vc += nr;
            if (!e_max_out || ch.nnz_rows == 0) continue;
            const uint32_t* rp = L.meta.data() + ch.meta_off + round_up4(ch.nnz_rows);
            if (nr == 1) { best = std::max(best, rp[ch.nnz_rows]); continue; }  // an uncut chunk: all its entries
            const uint32_t width = (ch.n_cols + nr - 1) / nr;
            cnt.assign(nr, 0u);
            const ChunkEntry* en = L.entries.data() + ch.ent_off;
            for (uint32_t i = 0; i < rp[ch.nnz_rows]; ++i) ++cnt[std::min(en[i].col_offset / width, nr - 1)];
            for (uint32_t v : cnt) best = std::max(best, v);
        }
        if (vc_ptr_out) (*vc_ptr_out)[L.n_chunks] = n_vc;
        if (e_max_out) *e_max_out = best;
        return n_vc;
    };
    const uint32_t fm_words = static_cast<uint32_t>((static_cast<uint64_t>(L.w_rows) + 31) / 32);
    CmLayout out;
    const uint32_t n_real = layout_for_cap(std::max<uint32_t>(L.c_max, 1u), nullptr, nullptr);
    for (uint32_t cap = std::max<uint32_t>(L.c_max, 1u); n_real > 0; cap = cap * 7 / 8) {
        uint32_t e_cap = 0;
        const uint32_t n_vc = layout_for_cap(cap, nullptr, &e_cap);
        if (static_cast<uint64_t>(n_vc) * 100u > static_cast<uint64_t>(n_real) * kCmMaxDup) break;
        const CmShape cand = cm_shape(fm_words, L.w_rows, L.r_max, e_cap, cap, L.n_chunks, n_vc);
        if (cand.ok) { out.shape = cand; break; }
        if (cap < 8u) break;
    }
    if (out.shape.ok) layout_for_cap(out.shape.col_cap, &out.vc_ptr, nullptr);
    return out;
}

// Whether layers 0 and 1 have the structure the prefix launch needs (their merged layer is build_prefix_layer's): layer 0 is
// one chunk of 1 .. kCmPrefixTop0 columns, each the parent of one layer-1 chunk; neither layer is rearranged or index-sharded;
// both share a feature space small enough for a direct table and the bias; the merged chunk has at most 256 columns.
inline bool prefix_mergeable(const ChunkedLayerHost& H0, const ChunkedLayerHost& H1) {
    const auto absent = [](const ChunkHeader& ch) { return (ch.has_bias & kChunkAbsent) != 0; };
    return H0.n_chunks == 1 && H0.n_cols >= 1 && H0.n_cols <= kCmPrefixTop0 && H1.n_chunks == H0.n_cols && !H0.reordered &&
           !H1.reordered && H0.w_rows == H1.w_rows && H0.w_rows <= kCmDirectRows &&
           std::memcmp(&H0.bias, &H1.bias, sizeof(float)) == 0 && H0.n_cols + H1.n_cols <= 256u &&
           std::none_of(H0.chunks.begin(), H0.chunks.end(), absent) && std::none_of(H1.chunks.begin(), H1.chunks.end(), absent);
}

// force: take the kernel wherever the layer has images, ignoring the reuse / occupancy heuristics (kernel mode 5, tests)
inline CmPlan cm_plan(const CmShape& s, uint32_t n_chunks, uint64_t pairs, uint32_t n_sm, bool force) {
    CmPlan p;
    if (!s.ok || pairs == 0) return p;
    // with the 94 KB feature-map image of a large feature space the kernel does not beat the query-major kernels (S layers
    // 1-4) -- only direct-table layers take it by default
    if (!force && !s.direct) return p;
    pairs = pairs * s.n_vc / std::max<uint32_t>(n_chunks, 1u);  // cut chunks are visited once per column range
    n_chunks = s.n_vc;
    if (!force && (pairs < static_cast<uint64_t>(kCmMinReuse) * n_chunks || pairs < static_cast<uint64_t>(kCmMinPairsPerSm) * n_sm)) return p;
    const size_t per_warp = cm_warp_bytes(s.acc_cols, s.stages);
    uint32_t warps = static_cast<uint32_t>(std::min<size_t>(kCmMaxWarps, (kCmSmemBudget - s.img_bytes - 64) / per_warp));
    // no point in more lanes than a CTA's share of the pair list holds
    const uint64_t share = (pairs + n_sm - 1) / n_sm;
    while (warps > kCmMinWarps && static_cast<uint64_t>(warps - 1) * 32 >= share) --warps;
    p.eligible = true;
    p.warps = warps;
    p.grid = n_sm;
    p.smem = s.img_bytes + warps * per_warp + 64;
    return p;
}

__device__ __forceinline__ void cm_cp_async4(void* smem_dst, const void* gmem_src) {
    const uint32_t d = static_cast<uint32_t>(__cvta_generic_to_shared(smem_dst));
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cm_cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cm_cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

// bulk asynchronous copy global -> shared (TMA engine, non-tensor form; SASS UBLKCP) completing on an mbarrier
__device__ __forceinline__ void cm_mbar_init(uint32_t mbar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(mbar), "r"(count) : "memory");
}
__device__ __forceinline__ void cm_bulk_load(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t mbar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(dst_smem), "l"(src), "r"(bytes), "r"(mbar) : "memory");
}
__device__ __forceinline__ void cm_mbar_wait(uint32_t mbar, uint32_t parity) {
    uint32_t done = 0;
    do {
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(mbar), "r"(parity) : "memory");
    } while (!done);
}

// LOAD TIME: one CTA per VIRTUAL chunk (chunk p, column range h; S.vc_ptr[p] = first virtual chunk of chunk p) packs its image (see CmShape) from the layer's
// device arrays: the rows' entries whose column falls into the range (contiguous inside a row: entries are stored in
// ascending column order), columns re-based to the range.
__global__ void __launch_bounds__(256)
xl_cm_build_images_kernel(const LayerDev L, const CmShape S, unsigned char* __restrict__ images) {
    const uint32_t vc = blockIdx.x;
    uint32_t c;
    {
        uint32_t lo = 0, hi = L.n_chunks;  // largest c with vc_ptr[c] <= vc
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (S.vc_ptr[mid] <= vc) lo = mid; else hi = mid;
        }
        c = lo;
    }
    const uint32_t hh = vc - S.vc_ptr[c];
    const uint32_t n_ranges = S.vc_ptr[c + 1] - S.vc_ptr[c];
    const ChunkHeader h = L.chunks[c];
    unsigned char* img = images + static_cast<uint64_t>(vc) * S.img_bytes;
    uint32_t* hdr = reinterpret_cast<uint32_t*>(img);
    float* ew = reinterpret_cast<float*>(img + S.off_ew);
    unsigned char* ec = img + S.off_ec;
    for (uint32_t i = threadIdx.x; i < S.img_bytes / 4u; i += blockDim.x) reinterpret_cast<uint32_t*>(img)[i] = 0u;
    __syncthreads();
    if (h.has_bias & kChunkAbsent) return;
    if (n_ranges == 0) return;
    const uint32_t width = (h.n_cols + n_ranges - 1u) / n_ranges;  // columns per range of THIS chunk
    const uint32_t lo = hh * width;
    if (lo >= h.n_cols) return;                                    // empty range: no pair is ever bucketed here
    const uint32_t hi = min(h.n_cols, lo + width);
    const uint32_t R = h.nnz_rows;
    const uint32_t R4 = (R + 3u) & ~3u;
    const uint32_t* ridx = L.meta + h.meta_off;
    const uint32_t* rp = ridx + R4;
    const uint2* ent = L.entries + h.ent_off;
    unsigned short* rps = S.direct ? nullptr : reinterpret_cast<unsigned short*>(img + S.off_rp);
    if (!S.direct) {
        uint32_t* lookup = reinterpret_cast<uint32_t*>(img + S.off_lookup);
        unsigned short* pre = reinterpret_cast<unsigned short*>(img + S.off_pre);
        const uint2* fm = L.featmap + static_cast<uint64_t>(c) * L.fm_words;
        for (uint32_t i = threadIdx.x; i < S.words; i += blockDim.x) {
            const uint2 cell = fm[i];
            lookup[i] = cell.x;
            pre[i] = static_cast<unsigned short>(cell.y);
        }
    }
    // rows in blocks of 256: sub-range of the row inside [lo, hi), exclusive scan of the lengths, copy
    __shared__ uint32_t s_scan[256];
    __shared__ uint32_t s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (uint32_t r0 = 0; r0 < R; r0 += 256u) {
        const uint32_t r = r0 + threadIdx.x;
        uint32_t b = 0, e = 0;
        if (r < R) {
            b = rp[r];
            e = rp[r + 1];
            while (b < e && ent[b].x < lo) ++b;
            uint32_t t = b;
            while (t < e && ent[t].x < hi) ++t;
            e = t;
        }
        const uint32_t len = e - b;
        s_scan[threadIdx.x] = len;
        __syncthreads();
        for (uint32_t d = 1; d < 256u; d <<= 1) {  // Hillis-Steele inclusive scan
            const uint32_t v = (threadIdx.x >= d) ? s_scan[threadIdx.x - d] : 0u;
            __syncthreads();
            s_scan[threadIdx.x] += v;
            __syncthreads();
        }
        const uint32_t base = s_carry + s_scan[threadIdx.x] - len;
        if (r < R) {
            for (uint32_t i = 0; i < len; ++i) {
                const uint2 en = ent[b + i];
                ec[base + i] = static_cast<unsigned char>(en.x - lo);
                ew[base + i] = __uint_as_float(en.y);
            }
            if (S.direct) {
                // start table: row r starts every feature after the previous row's up to its own (a feature without a row
                // reads as an empty range, as does a row without entries in this column range); the last row's end
                // closes the table at T[w_rows].  Rows ascend by feature.
                unsigned short* starts = reinterpret_cast<unsigned short*>(img + S.off_lookup);
                const uint32_t w_rows = S.words - 1u;
                const uint32_t f = min(ridx[r], w_rows);
                for (uint32_t g = r ? min(ridx[r - 1], w_rows) + 1u : 0u; g <= f; ++g) starts[g] = static_cast<unsigned short>(base);
                if (r + 1u == R)
                    for (uint32_t g = f + 1u; g <= w_rows; ++g) starts[g] = static_cast<unsigned short>(base + len);
            } else {
                rps[r] = static_cast<unsigned short>(base);
            }
            if (r + 1u == R) {
                if (!S.direct) rps[R] = static_cast<unsigned short>(base + len);
                hdr[0] = (h.has_bias & 1u) ? (base | ((base + len) << 16)) : 0u;  // the bias row is the chunk's last row
                hdr[3] = base + len;
            }
        }
        __syncthreads();
        if (threadIdx.x == 255u) s_carry += s_scan[255];
        __syncthreads();
    }
    if (threadIdx.x == 0) {
        hdr[1] = hi - lo;
        hdr[2] = R;
    }
}

// Bucketing (count -> scan -> scatter).  Every pair of a layer lands in its virtual chunk's bucket, and tens of thousands
// of pairs land on a few dozen chunks (eurlex-4k leaf: 154,490 pairs on 64; a layer-0 of one chunk: every query's pair on
// one).  Atomics on one counter serialise in the L2, so the pairs are counted per CTA in a shared-memory histogram and
// each CTA adds a non-empty bin to the global counter once.  A CTA walks a contiguous block of queries, one warp per query.
// The histogram covers kCmBinWindow virtual chunks at a time; a layer with more makes one pass over the CTA's queries per
// window, so shared memory stays bounded for any layer and any beam width.
constexpr uint32_t kCmBinWindow = 8192;     // virtual chunks one bucketing pass histograms (32 KB of shared memory)
constexpr int kCmBucketThreads = 1024;
constexpr uint32_t kCmBucketCtasPerSm = 2;  // 64 warps per SM; one CTA per SM took 2.4 us longer on the eurlex-4k leaf

// a CTA adds each of its bins once: few CTAs, few atomics on the same counter; at least one query per warp
inline uint32_t cm_bucket_grid(uint32_t rows, uint32_t n_sm) {
    return std::max(1u, std::min(kCmBucketCtasPerSm * n_sm, (rows + kCmBucketThreads / 32 - 1) / (kCmBucketThreads / 32)));
}

// the virtual chunks [lo, hi) of a beam slot on chunk p that fall into the bin window [b0, b0 + nb): one per non-empty
// column range of a scored chunk (cw columns each, range v - v0 starts at column (v - v0) x cw); none for an absent or
// empty chunk
struct CmSlotRanges { uint32_t v0, lo, hi, cw; };
__device__ __forceinline__ CmSlotRanges cm_slot_ranges(const uint4 h, const uint32_t* __restrict__ vc_ptr, uint32_t p,
                                                       uint32_t b0, uint32_t nb) {
    CmSlotRanges s{0, 0, 0, 0};
    if ((h.w & kChunkAbsent) || h.y == 0) return s;
    const uint32_t v0 = vc_ptr[p], nr = vc_ptr[p + 1] - v0;
    if (nr == 0) return s;
    s.v0 = v0;
    s.cw = (h.y + nr - 1u) / nr;
    const uint32_t n = min(nr, (h.y + s.cw - 1u) / s.cw);
    s.lo = max(v0, b0);
    s.hi = max(s.lo, min(v0 + n, b0 + nb));
    return s;
}

// queries [q_begin, q_end) of this CTA
__device__ __forceinline__ uint2 cm_bucket_block(uint32_t rows) {
    const uint32_t per = (rows + gridDim.x - 1) / gridDim.x;
    const uint32_t b = min(rows, blockIdx.x * per);
    return make_uint2(b, min(rows, b + per));
}

// candidate position of every beam slot (prefix of the chunk widths; first window) and pairs per virtual chunk
__global__ void __launch_bounds__(kCmBucketThreads, kCmBucketCtasPerSm)
xl_cm_count_kernel(const LayerDev L, const uint32_t* __restrict__ beam_id, const uint32_t* __restrict__ beam_cnt,
                   const uint32_t beam_stride, const uint32_t rows, CmWork w, const uint32_t* __restrict__ vc_ptr,
                   const uint32_t n_vc) {
    __shared__ uint32_t bins[kCmBinWindow];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
    const uint2 blk = cm_bucket_block(rows);
    for (uint32_t b0 = 0; b0 < n_vc; b0 += kCmBinWindow) {
        const uint32_t nb = min(kCmBinWindow, n_vc - b0);
        for (uint32_t i = threadIdx.x; i < nb; i += blockDim.x) bins[i] = 0u;
        __syncthreads();
        for (uint32_t q = blk.x + warp; q < blk.y; q += warps) {
            const uint32_t cnt = beam_cnt[q];
            uint32_t run = 0;
            for (uint32_t j0 = 0; j0 < cnt; j0 += 32) {
                const uint32_t j = j0 + lane;
                uint4 h = make_uint4(0, 0, 0, kChunkAbsent);  // {col_begin, n_cols, nnz_rows, has_bias}
                uint32_t p = 0;
                if (j < cnt) {
                    p = beam_id[static_cast<uint64_t>(q) * beam_stride + j];
                    h = *reinterpret_cast<const uint4*>(&L.chunks[p]);
                }
                if (b0 == 0) {
                    const uint32_t width = (j < cnt) ? h.y : 0u;
                    const uint32_t incl = warp_incl_scan(width, lane);
                    if (j < cnt) w.slot_pos[static_cast<uint64_t>(q) * beam_stride + j] = run + incl - width;
                    run += __shfl_sync(kFull, incl, 31);
                }
                const CmSlotRanges s = cm_slot_ranges(h, vc_ptr, p, b0, nb);
                for (uint32_t v = s.lo; v < s.hi; ++v) atomicAdd(&bins[v - b0], 1u);
            }
        }
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < nb; i += blockDim.x)
            if (bins[i]) atomicAdd(&w.count[b0 + i], bins[i]);
        __syncthreads();
    }
}

// Estimated work of one pair of a (virtual) chunk with E entries in a feature space of D rows: a pair looks up each of its
// query's features (about nnz shared-memory lookups) and adds the entries of the rows it hits (about nnz x E / D), so its
// cost is proportional to D + E -- one lookup weighs about as much as one entry (both are a few scattered shared-memory
// accesses).  The accumulate phase dominates on wide chunks, so pairs of an 84-column chunk cost ~1.3x those of a 62-column one.
__device__ __forceinline__ uint32_t cm_pair_cost(uint32_t w_rows, uint32_t entries) { return w_rows + entries; }

__device__ __forceinline__ uint64_t warp_incl_scan64(uint64_t v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint64_t t = __shfl_up_sync(kFull, v, d);
        if (lane >= d) v += t;
    }
    return v;
}

// single CTA: exclusive scans of the pair counts (bucket offsets) and of the chunks' estimated work (cost_ptr); count[]
// becomes the scatter cursor and claim[] the score kernel's claim cursor; active[] starts at 0.  A chunk's entry count is
// read from its image header.
__global__ void __launch_bounds__(1024)
xl_cm_scan_kernel(const uint32_t n_chunks, CmWork w, const unsigned char* __restrict__ images, const uint32_t img_bytes,
                  const uint32_t w_rows) {
    __shared__ uint32_t s_pairs[32];
    __shared__ uint64_t s_cost[32];
    __shared__ uint32_t carry_pairs;
    __shared__ uint64_t carry_cost;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    if (threadIdx.x == 0) { carry_pairs = 0; carry_cost = 0; }
    __syncthreads();
    for (uint32_t c0 = 0; c0 < n_chunks; c0 += 1024) {
        const uint32_t c = c0 + threadIdx.x;
        const uint32_t n = (c < n_chunks) ? w.count[c] : 0u;
        const uint32_t unit = n ? cm_pair_cost(w_rows, reinterpret_cast<const uint32_t*>(images + static_cast<uint64_t>(c) * img_bytes)[3]) : 1u;
        const uint64_t cost = static_cast<uint64_t>(n) * unit;
        const uint32_t in_p = warp_incl_scan(n, lane);
        const uint64_t in_c = warp_incl_scan64(cost, lane);
        if (lane == 31) { s_pairs[warp] = in_p; s_cost[warp] = in_c; }
        __syncthreads();
        if (warp == 0) {
            const uint32_t a = s_pairs[lane];
            const uint64_t b = s_cost[lane];
            const uint32_t ia = warp_incl_scan(a, lane);
            const uint64_t ib = warp_incl_scan64(b, lane);
            s_pairs[lane] = ia - a;
            s_cost[lane] = ib - b;
        }
        __syncthreads();
        const uint32_t ex_p = carry_pairs + s_pairs[warp] + in_p - n;
        const uint64_t ex_c = carry_cost + s_cost[warp] + in_c - cost;
        if (c < n_chunks) {
            w.bucket_ptr[c] = ex_p;
            w.cost_ptr[c] = ex_c;
            w.count[c] = ex_p;  // cursor
            w.claim[c] = ex_p;
            w.active[c] = 0;
        }
        __syncthreads();
        if (threadIdx.x == 1023) { carry_pairs = ex_p + n; carry_cost = ex_c + cost; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { w.bucket_ptr[n_chunks] = carry_pairs; w.cost_ptr[n_chunks] = carry_cost; }
}

// appends (query, candidate position) to the bucket of every virtual chunk a beam slot is scored on.  Per bin window a
// CTA counts its pairs per virtual chunk, reserves one contiguous run of each non-empty bucket (one atomic on its cursor),
// and places each pair at the run's next free place, counted by a shared-memory atomic; the bins hold the counts, then the
// CTA's cursors, so shared memory stays at one window at any beam width.  The order inside a bucket is free: a pair's
// result location is fixed by its query and position.
__global__ void __launch_bounds__(kCmBucketThreads, kCmBucketCtasPerSm)
xl_cm_scatter_kernel(const LayerDev L, const uint32_t* __restrict__ beam_id, const uint32_t* __restrict__ beam_cnt,
                     const uint32_t beam_stride, const uint32_t rows, CmWork w, const uint32_t* __restrict__ vc_ptr,
                     const uint32_t n_vc) {
    __shared__ uint32_t bins[kCmBinWindow];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
    const uint2 blk = cm_bucket_block(rows);
    for (uint32_t b0 = 0; b0 < n_vc; b0 += kCmBinWindow) {
        const uint32_t nb = min(kCmBinWindow, n_vc - b0);
        auto each_pair = [&](auto visit) {
            for (uint32_t q = blk.x + warp; q < blk.y; q += warps) {
                const uint32_t cnt = beam_cnt[q];
                for (uint32_t j = lane; j < cnt; j += 32) {
                    const uint32_t p = beam_id[static_cast<uint64_t>(q) * beam_stride + j];
                    const CmSlotRanges s = cm_slot_ranges(*reinterpret_cast<const uint4*>(&L.chunks[p]), vc_ptr, p, b0, nb);
                    if (s.lo < s.hi) visit(q, j, s);
                }
            }
        };
        for (uint32_t i = threadIdx.x; i < nb; i += blockDim.x) bins[i] = 0u;
        __syncthreads();
        each_pair([&](uint32_t, uint32_t, const CmSlotRanges& s) {
            for (uint32_t v = s.lo; v < s.hi; ++v) atomicAdd(&bins[v - b0], 1u);
        });
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < nb; i += blockDim.x)
            if (bins[i]) bins[i] = atomicAdd(&w.count[b0 + i], bins[i]);
        __syncthreads();
        each_pair([&](uint32_t q, uint32_t j, const CmSlotRanges& s) {
            const uint32_t pos = w.slot_pos[static_cast<uint64_t>(q) * beam_stride + j];
            for (uint32_t v = s.lo; v < s.hi; ++v) {
                const uint32_t at = atomicAdd(&bins[v - b0], 1u);
                w.pair_q[at] = q;
                w.pair_pos[at] = pos + (v - s.v0) * s.cw;  // first candidate of this column range
            }
        });
        __syncthreads();
    }
}

// The (virtual) chunk CTA b of `shares` starts on: the one where share b begins when the chunk-sorted pair list is cut into
// shares of equal estimated work (cost_ptr), so the CTAs start spread over the chunks in proportion to their work.
// n_vc: no pairs at all.
__device__ inline uint32_t cm_start_chunk(const CmWork& w, uint32_t n_vc, uint32_t b, uint32_t shares) {
    const uint64_t T = w.cost_ptr[n_vc];
    if (T == 0) return n_vc;
    const uint64_t t = static_cast<uint64_t>(T / shares) * b + (T % shares) * b / shares;  // floor(T * b / shares) < T without overflow
    uint32_t lo = 0, hi = n_vc;  // largest c with cost_ptr[c] <= t: a non-empty chunk, as cost_ptr[c + 1] > t
    while (hi - lo > 1) {
        const uint32_t mid = (lo + hi) >> 1;
        if (w.cost_ptr[mid] <= t) lo = mid; else hi = mid;
    }
    return lo;
}

// Diagnostics: built with -DPB200_CM_TRACE (tools/profile_cm_kernel.py) the score kernel records, for its last launch, every
// CTA's %globaltimer start / end and images staged, every warp's clock64 cycles by phase, its accumulate trips and useful
// slots (entries added; a trip offers 32 x kCmSlots), and the slices and pairs it scored, in g_cm_trace:
//   [0] grid, [1] warps per CTA, [2] pairs of the launch, then per CTA: start ns, end ns, images staged,
//   kCmMaxWarps x (kCmPhases cycles, trips, useful slots, slices, pairs).
// A chunk switch is two phases: the barrier with the choice of the next chunk, and the wait for the bulk copy.
// Without the define CmTrace is empty and the kernel is unchanged.
enum { kCmPhSwitch, kCmPhCopy, kCmPhStaging, kCmPhLookup, kCmPhAccumulate, kCmPhSlice, kCmPhases };
#ifdef PB200_CM_TRACE
constexpr uint32_t kCmTraceCtas = 1024;
constexpr uint32_t kCmTraceWarp = kCmPhases + 4;
constexpr uint32_t kCmTraceCta = 3 + kCmMaxWarps * kCmTraceWarp;
__device__ unsigned long long g_cm_trace[3 + kCmTraceCtas * kCmTraceCta];
__device__ __forceinline__ unsigned long long cm_globaltimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
struct CmTrace {
    unsigned long long start;
    long long t, ph[kCmPhases];
    unsigned long long trips, slots;  // trips: warp-uniform; slots: this lane's
    unsigned long long slices, pairs, images;  // slices, pairs: warp-uniform; images: CTA-uniform
    __device__ void begin() {
        start = cm_globaltimer();
        t = clock64();
        for (int p = 0; p < kCmPhases; ++p) ph[p] = 0;
        trips = slots = slices = pairs = images = 0;
    }
    __device__ void slice(uint32_t n_pairs) {
        ++slices;
        pairs += n_pairs;
    }
    __device__ void staged() { ++images; }
    __device__ void mark(int p) {
        const long long n = clock64();
        ph[p] += n - t;
        t = n;
    }
    __device__ void count(uint32_t n_trips, uint32_t n_slots) {
        trips += n_trips;
        slots += n_slots;
    }
    __device__ void flush(int warp, int lane, uint32_t launch_pairs) {  // every thread of the CTA calls it once, last
        __syncthreads();
        if (blockIdx.x >= kCmTraceCtas) return;
        unsigned long long* rec = g_cm_trace + 3 + blockIdx.x * kCmTraceCta;
        if (threadIdx.x == 0) {
            if (blockIdx.x == 0) { g_cm_trace[0] = gridDim.x; g_cm_trace[1] = blockDim.x >> 5; g_cm_trace[2] = launch_pairs; }
            rec[0] = start;
            rec[1] = cm_globaltimer();
            rec[2] = images;
        }
        for (int d = 16; d > 0; d >>= 1) slots += __shfl_xor_sync(kFull, slots, d);
        if (lane == 0) {
            unsigned long long* wr = rec + 3 + warp * kCmTraceWarp;
            for (int p = 0; p < kCmPhases; ++p) wr[p] = static_cast<unsigned long long>(ph[p]);
            wr[kCmPhases] = trips;
            wr[kCmPhases + 1] = slots;
            wr[kCmPhases + 2] = slices;
            wr[kCmPhases + 3] = pairs;
        }
    }
};
#else
struct CmTrace {
    __device__ void begin() {}
    __device__ void mark(int) {}
    __device__ void count(uint32_t, uint32_t) {}
    __device__ void slice(uint32_t) {}
    __device__ void staged() {}
    __device__ void flush(int, int, uint32_t) {}
};
#endif

// PREFIX: see CmPrefixOut (w, cand and cand_stride_q are unused; a CTA takes an equal slice of the tile's rows and stages the
// one image once).  Otherwise P is unused.
template <bool DIRECT, int STAGES, bool PREFIX = false>
__global__ void __launch_bounds__(kCmMaxWarps * 32, 1)
xl_cm_scores_kernel(const LayerDev L, const QueryDev X, const CmWork w, const CmShape S, const unsigned char* __restrict__ images,
                    float* __restrict__ cand, const uint64_t cand_stride_q, const CmPrefixOut P) {
    extern __shared__ __align__(128) unsigned char smem_raw[];
    unsigned char* img = smem_raw;                                   // the staged image of one virtual chunk
    // the image is only ever written by the bulk copy (async proxy), never by this kernel's stores: __restrict__ lets the
    // compiler hoist its loads above the accumulator stores
    const uint32_t* __restrict__ hdr_s = reinterpret_cast<const uint32_t*>(img);
    const unsigned short* __restrict__ start_s = reinterpret_cast<const unsigned short*>(img + S.off_lookup);  // direct: row starts
    const uint32_t* __restrict__ look_s = reinterpret_cast<const uint32_t*>(img + S.off_lookup);   // else feature-map bits
    const unsigned short* __restrict__ pre_s = reinterpret_cast<const unsigned short*>(img + S.off_pre);
    const unsigned short* __restrict__ rp_s = reinterpret_cast<const unsigned short*>(img + S.off_rp);
    const float* __restrict__ ew_s = reinterpret_cast<const float*>(img + S.off_ew);
    const unsigned char* __restrict__ ec_s = img + S.off_ec;
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int nwarps = blockDim.x >> 5;
    constexpr int kStride = kCmFeat + 1;
    constexpr int kBuf = 32 * kStride;                               // words per staging array
    constexpr int kNBuf = static_cast<int>(cm_buffers(STAGES));
    unsigned char* mine = smem_raw + S.img_bytes + static_cast<size_t>(warp) * cm_warp_bytes(S.acc_cols, STAGES);
    uint32_t* st_idx = reinterpret_cast<uint32_t*>(mine);            // [kNBuf][32][kStride]
    float* st_val = reinterpret_cast<float*>(st_idx + kNBuf * kBuf); // [kNBuf][32][kStride]
    float* my_acc = st_val + kNBuf * kBuf + lane;                    // [acc_cols][32], this lane's column of it

    __shared__ __align__(8) unsigned long long s_mbar;
    const uint32_t mbar = static_cast<uint32_t>(__cvta_generic_to_shared(&s_mbar));
    if (threadIdx.x == 0) {
        cm_mbar_init(mbar, 1u);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    }
    __syncthreads();
    CmTrace trace;
    trace.begin();

    // staging geometry: one warp-wide cp.async instruction copies kCmFeat consecutive features of kPerIter pairs; this lane
    // always serves feature fl of the pairs sub, sub + kPerIter, ...
    constexpr int kPerIter = 32 / kCmFeat;
    constexpr int kIters = 32 / kPerIter;
    const int sub = lane / kCmFeat, fl = lane % kCmFeat;
    uint32_t parity = 0;

    // The accumulate phase.  A lane's hit rows (entry ranges with their x, in feature order) are ONE stream of entries,
    // kCmSlots per trip whatever the rows' lengths, and the stream runs across rounds: after round r's lookup the warp runs
    // just enough trips for every lane to finish round r - 1's hits, and a lane that finishes early goes straight on into
    // round r's.  So the trip count follows the largest BACKLOG of a lane (entries looked up but not yet added), not each
    // round's busiest lane; one drain after the last round (with the bias row) runs to the busiest lane.  Slots of one trip
    // may hold entries of different rows, or a column a non-canonical row repeats: a slot whose column an earlier slot of
    // the trip also adds to starts from that slot's sum instead of the loaded accumulator, and the stores go out in slot
    // order -- every column sees exactly the sequential additions, in feature order (inference.hpp:788-811).
    //
    // Stream state, carried from round to round: the current row's entries [e, ee) with factor x; hp, the next hit to
    // take (a word offset in st_idx / st_val), loaded ahead into next_r / next_x; l1_end, one past the previous round's
    // last hit.  The previous round's hits and the newest round's are read as one list: hp jumps from l1_end to the newest
    // row.  Two rounds of hits are resident at once, hence the extra staging buffer (cm_buffers).  backlog: entries looked
    // up but not yet added.
    uint32_t e = 0, ee = 0, backlog = 0;
    float x = 0.0f;
    uint32_t hp = 0, l1_end = 0;  // word offsets in st_idx (and st_val)
    // row / cnt / n_ent: the newest round's compacted hits (its row in st_idx; the x sit at the same place in st_val),
    // their count and entries.  drain: run until every lane has added all of them, else only until every lane has
    // finished the previous round's.
    auto add_rows = [&](uint32_t row, uint32_t cnt, uint32_t n_ent, bool drain) {
        const uint32_t l2_end = row + cnt;
        const uint32_t avail = backlog + n_ent;
        const uint32_t trips = __reduce_max_sync(kFull, ((drain ? avail : backlog) + kCmSlots - 1u) / kCmSlots);
        if (hp == l1_end) hp = row;
        // the next row's range and x, loaded ahead of their use (read one past the last hit: the stride-9 row's spare word)
        uint32_t next_r = st_idx[hp];
        float next_x = st_val[hp];
        for (uint32_t t = 0; t < trips; ++t) {
            uint32_t es[kCmSlots], cs[kCmSlots];
            float xs[kCmSlots], a[kCmSlots];
            bool on[kCmSlots];  // true for a prefix of the slots
#pragma unroll
            for (int u = 0; u < kCmSlots; ++u) {
                if (e == ee && hp != l2_end) {
                    e = next_r & 0xFFFFu;
                    ee = next_r >> 16;
                    x = next_x;
                    ++hp;
                    if (hp == l1_end) hp = row;
                    next_r = st_idx[hp];
                    next_x = st_val[hp];
                }
                on[u] = e < ee;
                es[u] = e;  // an idle slot (only once the lane's backlog is all added) reads a valid, unused entry
                xs[u] = x;
                e += on[u] ? 1u : 0u;
            }
#pragma unroll
            for (int u = 0; u < kCmSlots; ++u) cs[u] = ec_s[es[u]];
#pragma unroll
            for (int u = 0; u < kCmSlots; ++u) a[u] = my_acc[cs[u] * 32u];
#pragma unroll
            for (int u = 0; u < kCmSlots; ++u) {
                float sum = a[u];
#pragma unroll
                for (int p = 0; p < u; ++p) sum = (cs[p] == cs[u]) ? a[p] : sum;  // a[p] already holds slot p's sum
                a[u] = __fadd_rn(sum, __fmul_rn(xs[u], ew_s[es[u]]));
            }
#pragma unroll
            for (int u = 0; u < kCmSlots; ++u)
                if (on[u]) my_acc[cs[u] * 32u] = a[u];
        }
        // every slot of a trip adds an entry while the lane has one, so the previous round's hits are all added now
        const uint32_t added = min(avail, trips * kCmSlots);
        backlog = avail - added;
        trace.count(trips, added);
        l1_end = l2_end;
    };

    // ---- stage the image of virtual chunk c: ONE bulk copy (the caller has made sure every warp has left the previous image)
    uint32_t bias_range = 0, n_cols = 0;
    auto stage_image = [&](uint32_t c) {
        if (threadIdx.x == 0) cm_bulk_load(static_cast<uint32_t>(__cvta_generic_to_shared(img)), images + static_cast<uint64_t>(c) * S.img_bytes, S.img_bytes, mbar);
        cm_mbar_wait(mbar, parity);
        parity ^= 1u;
        trace.staged();
        trace.mark(kCmPhCopy);
        bias_range = hdr_s[0];
        n_cols = hdr_s[1];
    };

    // ---- one warp scores the pairs [s0, s_end) (at most 32, one per lane) of the staged chunk
    auto score_slice = [&](uint32_t s0, uint32_t s_end) {
        const uint32_t pidx = s0 + lane;
        const bool have = pidx < s_end;
        uint32_t q = 0, pos = 0, qn = 0;
        uint64_t qb = 0;
        if (have) {
            if constexpr (PREFIX) {
                q = pidx;
            } else {
                q = w.pair_q[pidx];
                pos = w.pair_pos[pidx];
            }
            qb = X.row_ptr[q] - X.nnz_base;
            qn = static_cast<uint32_t>(X.row_ptr[q + 1] - X.nnz_base - qb);
        }
        const uint32_t qn_max = __reduce_max_sync(kFull, qn);
        // the pairs this lane copies for: source pointers (feature fl of the pair's row) and row lengths, once per slice
        uint32_t src_o[kIters], src_n[kIters];  // offsets fit 32 bits: a tile of queries holds < 2^32 non-zeros
#pragma unroll
        for (int it = 0; it < kIters; ++it) {
            const int pi = it * kPerIter + sub;
            src_o[it] = static_cast<uint32_t>(__shfl_sync(kFull, qb, pi)) + fl;
            src_n[it] = __shfl_sync(kFull, qn, pi);
        }
        // query features travel global -> shared by cp.async through a ring of STAGES buffers: rounds r + 1 .. r + STAGES - 1
        // are in flight while round r is processed.  Row i of a buffer = the next kCmFeat features of the slice's pair i
        // (stride 9 words: the lane-per-row reads are bank-conflict free).  A (possibly empty) group is committed for every
        // round slot, so "all but the newest STAGES - 1 groups are complete" always means "round r has landed".
        auto stage_round = [&](uint32_t t0, int buf) {
            if (t0 < qn_max) {
                uint32_t* di = st_idx + buf * kBuf + sub * kStride + fl;
                float* dv = st_val + buf * kBuf + sub * kStride + fl;
#pragma unroll
                for (int it = 0; it < kIters; ++it) {
                    if (t0 + fl < src_n[it]) {
                        cm_cp_async4(di + it * kPerIter * kStride, X.col_idx + src_o[it] + t0);
                        cm_cp_async4(dv + it * kPerIter * kStride, X.val + src_o[it] + t0);
                    }
                }
            }
            cm_cp_async_commit();
        };
        __syncwarp();
#pragma unroll
        for (int st = 0; st < STAGES - 1; ++st) stage_round(static_cast<uint32_t>(st) * kCmFeat, st);
        for (uint32_t col = 0; col < n_cols; ++col) my_acc[col * 32] = 0.0f;
        trace.mark(kCmPhSlice);
        uint32_t prev_f = kCmEmpty;
        e = ee = backlog = 0;
        x = 0.0f;
        hp = l1_end = 0;
        int buf = 0;
        for (uint32_t t0 = 0; t0 < qn_max; t0 += kCmFeat, buf = (buf + 1 == kNBuf) ? 0 : buf + 1) {
            // refills the buffer of round r - 2, whose hits the previous round's trips finished
            stage_round(t0 + (STAGES - 1) * kCmFeat, (buf + STAGES - 1) % kNBuf);
            cm_cp_async_wait<STAGES - 1>();
            __syncwarp();
            trace.mark(kCmPhStaging);
            uint32_t* my_idx = st_idx + buf * kBuf + lane * kStride;
            float* my_val = st_val + buf * kBuf + lane * kStride;
            const uint32_t n_here = (qn > t0) ? min(static_cast<uint32_t>(kCmFeat), qn - t0) : 0u;
            // phase 1: look the features up -- all loads of the round are issued before the first store (eight independent
            // feature / lookup / value loads in flight per lane) -- then compact the hits IN PLACE as {entry range, x}
            uint32_t fq[kCmFeat], rq[kCmFeat];
            float xq[kCmFeat];
#pragma unroll
            for (int k = 0; k < kCmFeat; ++k) {
                fq[k] = (static_cast<uint32_t>(k) < n_here) ? my_idx[k] : kCmEmpty;
                xq[k] = my_val[k];
            }
#pragma unroll
            for (int k = 0; k < kCmFeat; ++k) {
                const uint32_t f = fq[k];
                const bool dup = (f == prev_f);  // a repeated column index only counts once (the first occurrence)
                if (static_cast<uint32_t>(k) < n_here) prev_f = f;
                uint32_t range = 0;
                if (static_cast<uint32_t>(k) < n_here && !dup && f < L.w_rows) {
                    if (DIRECT) {
                        range = static_cast<uint32_t>(start_s[f]) | (static_cast<uint32_t>(start_s[f + 1]) << 16);
                    } else {
                        const uint32_t word = look_s[f >> 5];
                        const uint32_t bit = f & 31u;
                        if ((word >> bit) & 1u) {
                            const uint32_t row = static_cast<uint32_t>(pre_s[f >> 5]) + __popc(word & ((1u << bit) - 1u));
                            range = static_cast<uint32_t>(rp_s[row]) | (static_cast<uint32_t>(rp_s[row + 1]) << 16);
                        }
                    }
                }
                rq[k] = range;
            }
            uint32_t cnt = 0, n_ent = 0;
#pragma unroll
            for (int k = 0; k < kCmFeat; ++k) {
                const uint32_t e0 = rq[k] & 0xFFFFu, e1 = rq[k] >> 16;
                if (e1 > e0) {
                    my_idx[cnt] = rq[k];
                    my_val[cnt] = xq[k];
                    ++cnt;
                    n_ent += e1 - e0;
                }
            }
            trace.mark(kCmPhLookup);
            // phase 2: the rest of the previous round's hit rows, then as much of this round's as the trips hold, in
            // feature order, into this lane's accumulators
            add_rows(static_cast<uint32_t>(buf * kBuf + lane * kStride), cnt, n_ent, false);
            trace.mark(kCmPhAccumulate);
            __syncwarp();
        }
        cm_cp_async_wait<0>();
        {  // drain, bias row last (inference.hpp:806-811): the bias row is the last "round", staged in the buffer after the
           // last round's (its hits are gone, and no copy is in flight any more)
            const uint32_t o = static_cast<uint32_t>(buf * kBuf + lane * kStride);
            const uint32_t b0 = bias_range & 0xFFFFu, b1 = bias_range >> 16;
            const bool live = have && b1 > b0;
            st_idx[o] = bias_range;
            st_val[o] = L.bias;
            add_rows(o, live ? 1u : 0u, live ? b1 - b0 : 0u, true);
        }
        trace.mark(kCmPhAccumulate);
        if (have) {
            if constexpr (PREFIX) {
                // layer 0 keeps all n0 candidates: its top-k is the descending order of their exact keys (unused keys
                // are 0 and sort last; a real key never is 0)
                unsigned long long key[kCmPrefixTop0];
#pragma unroll
                for (uint32_t j = 0; j < kCmPrefixTop0; ++j)
                    key[j] = j < P.n0 ? xl_exact_key(xl_transform(my_acc[j * 32], P.pp_kind, P.pp_p), j) : 0ull;
#pragma unroll
                for (uint32_t a = 1; a < kCmPrefixTop0; ++a)
#pragma unroll
                    for (uint32_t b = a; b > 0; --b)
                        if (key[b] > key[b - 1]) { const unsigned long long t = key[b]; key[b] = key[b - 1]; key[b - 1] = t; }
                // layer 1's beam slot r is the chunk of layer-0 rank r: its children's raw scores go to the next
                // positions of the candidate row, in column order
                const uint64_t o = static_cast<uint64_t>(q) * P.beam_stride;
                float* dst = P.cand1 + static_cast<uint64_t>(q) * P.cand1_stride;
#pragma unroll
                for (uint32_t r = 0; r < kCmPrefixTop0; ++r) {
                    if (r < P.n0) {
                        const uint32_t j = xl_exact_key_pos(key[r]);
                        P.beam_id[o + r] = j;
                        P.beam_val[o + r] = xl_exact_key_value(key[r]);
                        const ChunkHeader h = P.chunks1[j];
                        const float* src = my_acc + (P.n0 + h.col_begin) * 32u;
                        for (uint32_t col = 0; col < h.n_cols; ++col) dst[col] = src[col * 32];
                        dst += h.n_cols;
                    }
                }
                P.beam_cnt[q] = P.n0;
            }
        }
        if constexpr (!PREFIX) {
            // write-out, kCmFeat columns at a time through a [32][kStride] tile in the last round's buffer (free once the
            // drain is done; the next slice's first stage_round comes after a __syncwarp): lane i puts its pair's columns
            // into row i, then every store instruction writes kCmFeat consecutive columns of each of kPerIter pairs (the
            // staging geometry: this lane serves column fl of the pairs sub, sub + kPerIter, ...) where a store per column
            // touched 32 scattered candidate rows
            float* tile = st_val + ((buf + kNBuf - 1) % kNBuf) * kBuf;
            const uint32_t n_pairs = s_end - s0;
            const uint64_t o_mine = have ? static_cast<uint64_t>(q) * cand_stride_q + pos : 0u;
            float* dst[kIters];
#pragma unroll
            for (int it = 0; it < kIters; ++it) dst[it] = cand + __shfl_sync(kFull, o_mine, it * kPerIter + sub) + fl;
            for (uint32_t c0 = 0; c0 < n_cols; c0 += kCmFeat) {
                const uint32_t nc = min(static_cast<uint32_t>(kCmFeat), n_cols - c0);
                __syncwarp();
#pragma unroll
                for (int k = 0; k < kCmFeat; ++k)
                    if (static_cast<uint32_t>(k) < nc) tile[lane * kStride + k] = my_acc[(c0 + k) * 32];
                __syncwarp();
                if (static_cast<uint32_t>(fl) < nc) {
#pragma unroll
                    for (int it = 0; it < kIters; ++it)
                        if (static_cast<uint32_t>(it * kPerIter + sub) < n_pairs) dst[it][c0] = tile[(it * kPerIter + sub) * kStride + fl];
                }
            }
        }
        trace.slice(s_end - s0);
        trace.mark(kCmPhSlice);
    };

    if constexpr (PREFIX) {
        // every pair costs the same: equal slices of the rows, and warps take 32-pair slices of the CTA's
        const uint32_t begin = static_cast<uint32_t>(static_cast<uint64_t>(P.rows) * blockIdx.x / gridDim.x);
        const uint32_t end = static_cast<uint32_t>(static_cast<uint64_t>(P.rows) * (blockIdx.x + 1u) / gridDim.x);
        if (begin < end) {
            stage_image(0);
            for (uint32_t s0 = begin + static_cast<uint32_t>(warp) * 32u; s0 < end; s0 += static_cast<uint32_t>(nwarps) * 32u)
                score_slice(s0, min(s0 + 32u, end));
        }
        trace.flush(warp, lane, P.rows);
    } else {
        // Claim cursors decide which pairs this CTA scores, so the output cannot depend on the schedule: a pair's result
        // goes to the place its query and position fix.  The cursors and CTA counts are read back through L2 (__ldcg): the
        // claims of other SMs are atomics there, and a stale line in this SM's L1 could show a dry chunk as unclaimed
        // again and again.
        const uint32_t n_vc = S.n_vc;
        __shared__ unsigned long long s_pick_work[kCmMaxWarps];
        __shared__ uint32_t s_pick_act[kCmMaxWarps];
        __shared__ uint32_t s_pick_c[kCmMaxWarps];
        // the better of two candidates (unclaimed work, CTAs on the chunk, chunk): more work per CTA once this one joins,
        // work / (active + 1), compared crosswise (work < 2^32 pairs x 2^17, active <= grid: the products fit 64 bits),
        // then the lower index; n_vc = none.  CTAs that become free together spread over the chunks instead of all
        // draining the one with the most work and switching again.
        auto better = [n_vc](unsigned long long wa, uint32_t aa, uint32_t ca, unsigned long long wb, uint32_t ab, uint32_t cb) {
            if (ca == n_vc) return false;
            if (cb == n_vc) return true;
            const unsigned long long la = wa * (ab + 1u), lb = wb * (aa + 1u);
            return la > lb || (la == lb && ca < cb);
        };
        uint32_t c = cm_start_chunk(w, n_vc, blockIdx.x, gridDim.x);
        trace.mark(kCmPhSwitch);
        while (c < n_vc) {
            if (threadIdx.x == 0) atomicAdd(w.active + c, 1u);
            stage_image(c);
            const uint32_t c_end = w.bucket_ptr[c + 1];
            for (;;) {  // warps claim the chunk's slices until it runs dry
                uint32_t s0 = 0;
                if (lane == 0) s0 = atomicAdd(w.claim + c, 32u);
                s0 = __shfl_sync(kFull, s0, 0);
                if (s0 >= c_end) break;
                score_slice(s0, min(s0 + 32u, c_end));
            }
            // every warp has left the image: the CTA leaves the chunk and moves to the one with the most unclaimed
            // estimated work per CTA.  A cursor or count read here may already be stale; that only affects the choice, as
            // the claims themselves are atomic.
            __syncthreads();
            if (threadIdx.x == 0) atomicSub(w.active + c, 1u);
            unsigned long long bw = 0;
            uint32_t ba = 0, bc = n_vc;
            for (uint32_t v = threadIdx.x; v < n_vc; v += blockDim.x) {
                const uint32_t v_end = w.bucket_ptr[v + 1];
                const uint32_t cl = __ldcg(w.claim + v);
                if (cl >= v_end) continue;
                const uint32_t entries = reinterpret_cast<const uint32_t*>(images + static_cast<uint64_t>(v) * S.img_bytes)[3];
                const unsigned long long work = static_cast<unsigned long long>(v_end - cl) * cm_pair_cost(L.w_rows, entries);
                const uint32_t act = __ldcg(w.active + v);
                if (better(work, act, v, bw, ba, bc)) { bw = work; ba = act; bc = v; }
            }
            for (int d = 16; d > 0; d >>= 1) {
                const unsigned long long ow = __shfl_xor_sync(kFull, bw, d);
                const uint32_t oa = __shfl_xor_sync(kFull, ba, d);
                const uint32_t oc = __shfl_xor_sync(kFull, bc, d);
                if (better(ow, oa, oc, bw, ba, bc)) { bw = ow; ba = oa; bc = oc; }
            }
            if (lane == 0) { s_pick_work[warp] = bw; s_pick_act[warp] = ba; s_pick_c[warp] = bc; }
            __syncthreads();
            // s_pick_* are rewritten only after the next switch's first barrier, which every thread reaches after this read
            bw = s_pick_work[0];
            ba = s_pick_act[0];
            c = s_pick_c[0];
            for (int k = 1; k < nwarps; ++k)
                if (better(s_pick_work[k], s_pick_act[k], s_pick_c[k], bw, ba, c)) { bw = s_pick_work[k]; ba = s_pick_act[k]; c = s_pick_c[k]; }
            trace.mark(kCmPhSwitch);
        }
        trace.flush(warp, lane, w.bucket_ptr[n_vc]);
    }
}
