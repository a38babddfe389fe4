/* TEST INFRASTRUCTURE ONLY -- plain-C restatement of PairwiseANN::predict_single (pecos/core/ann/pairwise.hpp:265-288) as
 * driven by C_PAIRWISE_ANN_PREDICT (pecos/core/libpecos.cpp:628-657).
 *
 * Per pair b: query row (same ? 0 : b), column keys[b] of Y_csc.  Every column entry is pushed, in stored order, into a
 * max-heap keyed on distance only (KeyValPair::operator<); if topk < nnz the heap is popped down to topk; then sort_heap.
 * Slot k < heap size of row b receives {row id, distance, Y value, 1}; other slots are not written.
 * Distances: hno_distance / hno_sparse_distance of hnsw_oracle.c (the reference's FeatVec{Dense,Sparse}IPSimd::distance). */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

float hno_distance(const float* x, const float* y, uint32_t len, int metric, int isa);
float hno_sparse_distance(size_t s_a, const float* x, const uint32_t* A, size_t s_b, const float* y, const uint32_t* B, int metric,
                          int isa);

typedef struct {
    uint32_t idx;
    float dist;
    float val;
} pwo_pair_t;

/* libstdc++ __push_heap / __adjust_heap with std::less on the distance */
static void push_heap_(pwo_pair_t* first, long hole, long top, pwo_pair_t value) {
    long parent = (hole - 1) / 2;
    while (hole > top && first[parent].dist < value.dist) {
        first[hole] = first[parent];
        hole = parent;
        parent = (hole - 1) / 2;
    }
    first[hole] = value;
}

static void adjust_heap_(pwo_pair_t* first, long hole, long len, pwo_pair_t value) {
    const long top = hole;
    long child = hole;
    while (child < (len - 1) / 2) {
        child = 2 * (child + 1);
        if (first[child].dist < first[child - 1].dist) child--;
        first[hole] = first[child];
        hole = child;
    }
    if ((len & 1) == 0 && child == (len - 2) / 2) {
        child = 2 * (child + 1);
        first[hole] = first[child - 1];
        hole = child - 1;
    }
    push_heap_(first, hole, top, value);
}

static void pop_heap_(pwo_pair_t* h, long n) { /* std::pop_heap(h, h + n) */
    if (n > 1) {
        pwo_pair_t value = h[n - 1];
        h[n - 1] = h[0];
        adjust_heap_(h, 0, n - 1, value);
    }
}

/* sparse != 0: X rows / query rows are csr (x_ptr, x_idx, x_val / q_ptr, q_idx, q_val); else dense (x_val / q_val, d columns).
 * Returns 0, or 1 if a label key is out of range (nothing is written then). */
int pwo_predict(int sparse, int isa, uint32_t d, const uint64_t* x_ptr, const uint32_t* x_idx, const float* x_val, uint32_t num_label,
                const uint64_t* y_ptr, const uint32_t* y_idx, const float* y_val, const uint64_t* q_ptr, const uint32_t* q_idx,
                const float* q_val, uint32_t batch, uint32_t topk, const uint32_t* keys, int same, uint32_t* I, uint32_t* M, float* D,
                float* V) {
    uint64_t longest = 1;
    for (uint32_t b = 0; b < batch; ++b) {
        if (keys[b] >= num_label) return 1;
        if (y_ptr[keys[b] + 1] - y_ptr[keys[b]] > longest) longest = y_ptr[keys[b] + 1] - y_ptr[keys[b]];
    }
    pwo_pair_t* h = (pwo_pair_t*)malloc(sizeof(pwo_pair_t) * longest);
    for (uint32_t b = 0; b < batch; ++b) {
        const uint32_t q = same ? 0u : b;
        const uint64_t c0 = y_ptr[keys[b]], nnz = y_ptr[keys[b] + 1] - c0;
        long n = 0;
        for (uint64_t j = 0; j < nnz; ++j) {
            const uint32_t r = y_idx[c0 + j];
            pwo_pair_t v;
            v.idx = r;
            v.val = y_val[c0 + j];
            if (sparse)
                v.dist = hno_sparse_distance(q_ptr[q + 1] - q_ptr[q], q_val + q_ptr[q], q_idx + q_ptr[q], x_ptr[r + 1] - x_ptr[r],
                                             x_val + x_ptr[r], x_idx + x_ptr[r], 0, isa);
            else
                v.dist = hno_distance(q_val + (uint64_t)q * d, x_val + (uint64_t)r * d, d, 0, isa);
            h[n] = v;
            ++n;
            push_heap_(h, n - 1, 0, v);
        }
        if ((uint64_t)topk < nnz) {
            while (n > (long)topk) {
                pop_heap_(h, n);
                --n;
            }
        }
        for (long m = n; m > 1; --m) pop_heap_(h, m); /* std::sort_heap */
        for (long k = 0; k < n; ++k) {
            const uint64_t o = (uint64_t)b * topk + (uint64_t)k;
            I[o] = h[k].idx;
            D[o] = h[k].dist;
            V[o] = h[k].val;
            M[o] = 1u;
        }
    }
    free(h);
    return 0;
}
