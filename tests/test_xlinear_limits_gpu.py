"""GPU tests of XR-Linear prediction at the capacity limits that decide which score and top-k kernel runs for a layer, and
how a kernel splits its own work.  Every case puts one quantity on a limit and one past it, and then

* reads the kernel ids of the call (pb200_xlinear_get_kernel_ids) and asserts the kernel expected on each side of the
  edge, so the test fails if a threshold or its comparison moves;
* requires the same ids, counts and score bits from every kernel mode that runs on the shape;
* compares with the C restatement (oracle/restatement.py) and, where it is built, the reference library;
* checks every returned score against a float64 evaluation of the label's path (`_f64_check`), with a tolerance derived
  from the float32 accumulation bound, and for one-layer models also which labels made the top-k.

Score kernel ids: 0 row-list streaming, 1 feature-map lookup (warp per chunk), 2 dense queries, 3 query-warp, 4 chunk-major.
Top-k ids: 0 block sort, 1 warp select, 2 estimate filter.  Kernel modes (pb200_xlinear_set_lookup): 0 first generation
(row lists + block sort), 1 default, 2 no query-warp kernel, 3 query-warp wherever eligible, 4 no estimate filter,
5 chunk-major wherever it fits, 6 no chunk-major / prefix kernel, 7 no prefix kernel.

Candidate-row limits compare against cand_stride_q = b_prev x c_max (the beam entering the layer times its widest chunk),
not the real candidate count; only the block top-k's single-sort capacity (2048) compares against the valid candidates.

Limits considered but not reachable in a test, and so not tested here:
* the 2^32 feature-offset guard of the chunk-major kernel (rows x longest query >= 2^32);
* the 4 GiB cap on a staged tile of dense queries;
* the chunk-major image's e_max < 65535 check: an image with that many entries cannot fit 224 KB of shared memory anyway.
"""
import os
from ctypes import c_double, c_int, c_uint64

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .util import assert_csr_parity, random_tree

pytestmark = pytest.mark.gpu

U = 2.0 ** -24  # unit roundoff of float32


# ------------------------------------------------------------------------------------------------ model builders
def _weights(seed, n_cols, D, nnz_per_col, bias=1.0):
    return synth._random_weight_matrix(np.random.default_rng(seed), n_cols, D, nnz_per_col, bias)


def _flat_layers(seed, width, D, nnz_per_col):
    """One-layer model: a single chunk of `width` columns (b_prev = 1, cand_stride_q = width)."""
    W = _weights(seed, width, D, nnz_per_col)
    return [(W, smat.csc_matrix(np.ones((width, 1), dtype=np.float32)))]


def _two_layer(seed, widths, D, nnz_per_col, cover=None):
    """Layer 0: one chunk of len(widths) columns; layer 1: chunk j has widths[j] columns.  cover=R: every layer-1 chunk's
    rows are exactly the features [0, R) (feature r sits in the chunk's column r mod width, plus nnz_per_col random
    rows per column), so a query's matches in every chunk = its features below R, plus the bias row."""
    B = len(widths)
    W0 = _weights(seed, B, D, nnz_per_col)
    C0 = smat.csc_matrix(np.ones((B, 1), dtype=np.float32))
    C1 = synth._contiguous_codes(widths)
    if cover is None:
        return [(W0, C0), (_weights(seed + 1, int(sum(widths)), D, nnz_per_col), C1)]
    rng = np.random.default_rng(seed + 1)
    rows, cols = [], []
    c0 = 0
    for w in widths:
        r = np.arange(cover)
        rows.append(r)
        cols.append(c0 + r % w)
        extra = rng.integers(0, cover, size=(w, nnz_per_col))
        rows.append(extra.ravel())
        cols.append(np.repeat(np.arange(c0, c0 + w), nnz_per_col))
        c0 += w
    rows.append(np.full(c0, D))  # bias row
    cols.append(np.arange(c0))
    rows, cols = np.concatenate(rows), np.concatenate(cols)
    vals = rng.standard_normal(rows.size).astype(np.float32) * np.float32(0.3)
    vals[vals == 0] = np.float32(0.3)
    W1 = smat.coo_matrix((vals, (rows, cols)), shape=(D + 1, c0)).tocsc()
    W1.sum_duplicates()
    W1.sort_indices()
    return [(W0, C0), (W1.astype(np.float32), C1)]


def _exact_columns(seed, counts, D):
    """W (D + 1) x len(counts): column c holds counts[c] distinct random features and the bias row, so a chunk's entries
    are exactly sum(counts[c] + 1) over its columns."""
    rng = np.random.default_rng(seed)
    rows = [np.r_[np.sort(rng.choice(D, int(n), replace=False)), D] for n in counts]
    cols = np.repeat(np.arange(len(counts)), [r.size for r in rows])
    vals = (rng.standard_normal(cols.size) * 0.3).astype(np.float32)
    vals[vals == 0] = np.float32(0.3)
    W = smat.csc_matrix((vals, (np.concatenate(rows), cols)), shape=(D + 1, len(counts)))
    W.sort_indices()
    return W


def _spread(total, n):
    """n non-negative counts summing to `total`, as even as possible."""
    out = np.full(n, total // n, dtype=np.int64)
    out[: total - out.sum()] += 1
    return out


# Chunk-major image arithmetic of a direct-table layer (cm_shape, xlinear_cm_kernel.cuh).  An image is a 16-byte header,
# the table of u16 row starts (w_rows + 1 words), the entries' u32 weights and u8 column offsets (e_max + 1 each), every
# part padded to 16 bytes and the image to 128.  A warp takes (stages + 1) staging buffers of 32 x 9 x 8 bytes plus
# acc_cols x 32 x 4 bytes of accumulators (stages = 4 up to 16 columns, else 2).  The image fits when it leaves room for
# kCmMinWarps = 4 warps within kCmSmemBudget = 224 KB, less 64 bytes of CTA state.
CM_SMEM_BUDGET = 224 << 10
CM_MIN_WARPS = 4


def _a16(x):
    return (x + 15) // 16 * 16


def _cm_warp_bytes(acc_cols):
    stages = 4 if acc_cols <= 16 else 2
    return (stages + 1) * 32 * 9 * 8 + acc_cols * 32 * 4


def _cm_direct_image_bytes(w_rows, e_max):
    off = 16 + _a16((w_rows + 1) * 2) + _a16((e_max + 1) * 4) + _a16(e_max + 1)
    return (off + 127) // 128 * 128


def _cm_direct_fits(w_rows, e_max, acc_cols):
    return _cm_direct_image_bytes(w_rows, e_max) + CM_MIN_WARPS * _cm_warp_bytes(acc_cols) + 64 <= CM_SMEM_BUDGET


def _cm_max_entries(w_rows, acc_cols):
    """Most entries one direct-table image of acc_cols columns may hold (the next entry does not fit)."""
    lo, hi = 0, 65535
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if _cm_direct_fits(w_rows, mid, acc_cols) else (lo, mid)
    return lo


CAP_D, CAP_WIDTHS = 1000, [200] + [10] * 8  # leaf chunks; layer 0 has 9 columns, so the prefix launch stays out of it


def _cap_loop_layers(outside):
    """Leaf whose widest chunk (200 columns) holds the most entries an uncut image of 200 columns takes (W rows 1001), or
    one more.  Inside, the cap loop keeps cap = c_max = 200 and the 9 chunks stay whole.  Outside, the uncut image fails
    and the loop takes the next cap, 200 * 7 / 8 = 175: the widest chunk becomes two ranges of 100 columns, each with
    about half the entries, which fit (10 virtual chunks)."""
    e = _cm_max_entries(CAP_D + 1, 200) + (1 if outside else 0)
    counts = np.r_[_spread(e - 200, 200), np.full(80, 12)]
    W1 = _exact_columns(601, counts, CAP_D)
    W0 = _weights(602, len(CAP_WIDTHS), CAP_D, 20)
    return [(W0, smat.csc_matrix(np.ones((len(CAP_WIDTHS), 1), dtype=np.float32))),
            (W1, synth._contiguous_codes(CAP_WIDTHS))], e


PFX_D, PFX_N0, PFX_WIDTHS = 1000, 4, [15] * 4


def _prefix_budget_layers(outside):
    """Layers 0 (4 columns) and 1 (4 chunks of 15) whose merged prefix image (64 columns, W rows 1001) holds the most
    entries that fit next to 4 warps, or one more.  The merged entries are all of both layers' stored entries."""
    e = _cm_max_entries(PFX_D + 1, PFX_N0 + sum(PFX_WIDTHS)) + (1 if outside else 0)
    n = PFX_N0 + sum(PFX_WIDTHS)
    counts = _spread(e - n, n)
    W = _exact_columns(611, counts, PFX_D)
    W0, W1 = W[:, :PFX_N0], W[:, PFX_N0:]
    return [(smat.csc_matrix(W0), smat.csc_matrix(np.ones((PFX_N0, 1), dtype=np.float32))),
            (smat.csc_matrix(W1), synth._contiguous_codes(PFX_WIDTHS))], e


def _save(folder, layers, only_topk=10):
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=only_topk, skip_root_C=len(layers) == 1)
    return folder


def _queries(seed, D, nnz_list, cover=None, match_list=None):
    """CSR batch whose rows have the given numbers of features (sorted, distinct), followed by the rows every batch here
    holds: an empty row, a copy of row 0 and a copy of the longest row with one column index repeated (non-canonical: only
    the first occurrence counts).  cover / match_list: row i has exactly match_list[i] of its features below `cover`."""
    rng = np.random.default_rng(seed)
    rows = []
    for i, n in enumerate(nnz_list):
        if match_list is None:
            f = rng.choice(D, size=n, replace=False)
        else:
            m = match_list[i]
            f = np.concatenate([rng.choice(cover, size=m, replace=False), cover + rng.choice(D - cover, size=n - m, replace=False)])
        rows.append(np.sort(f))
    longest = int(np.argmax(nnz_list))
    rows.append(np.zeros(0, dtype=np.int64))
    rows.append(rows[0].copy())
    dup = rows[longest].copy()
    if dup.size > 2:
        dup[dup.size // 2] = dup[dup.size // 2 - 1]
    rows.append(dup)
    indptr = np.cumsum([0] + [r.size for r in rows])
    idx = np.concatenate(rows).astype(np.int64)
    vals = rng.uniform(0.05, 1.0, size=idx.size).astype(np.float32)
    X = smat.csr_matrix((vals, idx, indptr), shape=(len(rows), D))
    X.has_sorted_indices = True
    return X


def _dedup_first(X):
    """The query the reference scores: of a repeated column index only the first occurrence counts."""
    X = smat.csr_matrix(X)
    keep = np.ones(X.nnz, dtype=bool)
    for r in range(X.shape[0]):
        b, e = X.indptr[r], X.indptr[r + 1]
        keep[b + 1:e] = X.indices[b + 1:e] != X.indices[b:e - 1]
    rows = np.repeat(np.arange(X.shape[0]), np.diff(X.indptr))[keep]
    return smat.csr_matrix((X.data[keep].astype(np.float64), (rows, X.indices[keep])), shape=X.shape)


# ------------------------------------------------------------------------------------------------ float64 reference
def _pp(name):
    from oracle.restatement import parse_post_processor

    return parse_post_processor(name)


def _transform64(v, e, kind, p):
    """Post-processor of inference.hpp:208-238 in float64 at v, and a bound of its error when v is off by at most e: the
    largest |f'| over [v - e, v + e] times e, plus the roundings of the float32 steps (hinge base, result)."""
    lo, hi = v - e, v + e

    def f(x):
        if kind == 1:
            return 1.0 / (1.0 + np.exp(-x))
        if kind == 2:
            return -np.log1p(np.exp(-x))
        if kind in (3, 4):
            z = np.maximum(0.0, 1.0 - x) ** p if p > 0 else np.ones_like(x)
            return np.exp(-z) if kind == 3 else -z
        return x

    def df(x):
        if kind == 1:
            s = 1.0 / (1.0 + np.exp(-x))
            return s * (1.0 - s)
        if kind == 2:
            return 1.0 / (1.0 + np.exp(x))
        if kind in (3, 4):
            z = np.maximum(0.0, 1.0 - x)
            d = p * z ** (p - 1) if p > 0 else np.zeros_like(x)
            return d * (np.exp(-z ** p) if kind == 3 else 1.0)
        return np.ones_like(x)

    t = f(v)
    slope = np.maximum(np.maximum(np.abs(df(lo)), np.abs(df(hi))), np.abs(df(v)))
    if kind in (3, 4):
        # the hinge base is narrowed to float (relative U), z^p picks up p U of itself, the exponent's error passes into exp
        zp = np.maximum(0.0, 1.0 - np.minimum(lo, v)) ** max(p, 0)
        round_err = p * U * zp * (np.abs(t) if kind == 3 else 1.0) + 2 * U * np.abs(t)
    elif kind in (1, 2):
        round_err = 4 * U * (np.abs(t) + 1e-300) + (4 * U * np.exp(-v) / (1.0 + np.exp(-v)) if kind == 2 else 0.0)
    else:
        round_err = 0.0
    return t, slope * e + round_err


def _f64_scores(layers, bias, X, got, pp):
    """float64 value and error bound of every returned (query, label) score of `got` (csr) for the model `layers`
    ([(W, C)], W (D + 1) x n with the bias row last).

    Per layer on the label's path, raw = x . W[:, node] + bias * W[D, node] in float64, and the float32 kernel's raw score
    is within 2 n 2^-24 sum_i |x_i w_i| of it (n = the column's stored entries, an upper bound of the terms it adds).  That
    error is carried through the post-processor by its derivative (`_transform64`), then through the reference's combine
    rule (inference.hpp:208-238: sigmoid / lp-hinge multiply by the parent's value, log-sigmoid / log-lp-hinge add, noop
    keeps the layer's own value), each float32 combine adding one rounding.  Returns (value, bound) arrays aligned with
    got.data."""
    kind, p = _pp(pp)
    dense = not smat.issparse(X)
    Xq = smat.csr_matrix(np.asarray(X, dtype=np.float64)) if dense else _dedup_first(X)
    Xb = smat.hstack([Xq, smat.csr_matrix(np.full((Xq.shape[0], 1), bias))]).tocsr() if bias > 0 else Xq
    depth = len(layers)
    parents = []
    for d, (_, C) in enumerate(layers):
        Cr = smat.csr_matrix(C)
        parents.append(np.asarray([Cr.indices[Cr.indptr[i]] if Cr.indptr[i + 1] > Cr.indptr[i] else -1
                                   for i in range(Cr.shape[0])]))
    got = smat.csr_matrix(got)
    qs = np.repeat(np.arange(got.shape[0]), np.diff(got.indptr))
    nodes = np.asarray(got.indices, dtype=np.int64)
    val = None
    err = None
    # walk from the leaf up, collecting the node of every layer on each returned label's path
    path = [None] * depth
    path[depth - 1] = nodes
    for d in range(depth - 1, 0, -1):
        path[d - 1] = parents[d][path[d]]
    for d in range(depth):
        W = smat.csc_matrix(layers[d][0], dtype=np.float64)
        n_terms = np.diff(W.indptr)
        Wd = W[:, path[d]]  # one column per returned entry
        Xr = Xb[qs]
        raw = np.asarray(Xr.multiply(Wd.T).sum(axis=1)).ravel()
        mag = np.asarray(abs(Xr).multiply(abs(Wd).T).sum(axis=1)).ravel()
        e_raw = 2.0 * n_terms[path[d]] * U * mag + U * np.abs(raw)
        t, e_t = _transform64(raw, e_raw, kind, p)
        if d == 0 or kind == 0:
            val, err = t, e_t
        elif kind in (1, 3):
            nv = t * val
            err = np.abs(t) * err + np.abs(val) * e_t + e_t * err + U * np.abs(nv)
            val = nv
        else:
            nv = t + val
            err = err + e_t + U * np.abs(nv)
            val = nv
    return val, err


def _f64_check(layers, bias, X, got, pp, topk=None, what=""):
    """Every returned score lies within its bound of the float64 value.  For a one-layer model (topk given), also the
    membership: any label that the exact float64 top-k holds and the kernel left out, or the reverse, must score within
    the tolerance of the k-th float64 score."""
    val, err = _f64_scores(layers, bias, X, got, pp)
    g = np.asarray(smat.csr_matrix(got).data, dtype=np.float64)
    bad = np.abs(g - val) > err
    assert not bad.any(), (f"{what} {pp}: {int(bad.sum())} scores off their float64 value; first: got {g[bad][0]!r} "
                           f"want {val[bad][0]!r} +- {err[bad][0]:.3e}")
    if topk is None or len(layers) != 1:
        return
    got = smat.csr_matrix(got)
    all_lab = smat.csr_matrix(np.ones((X.shape[0], layers[0][0].shape[1]), dtype=np.float32))
    v_all, e_all = _f64_scores(layers, bias, X, all_lab, pp)
    n = layers[0][0].shape[1]
    v_all, e_all = v_all.reshape(-1, n), e_all.reshape(-1, n)
    for q in range(X.shape[0]):
        k = min(topk, n)
        order = np.argsort(-v_all[q], kind="stable")
        exact = set(order[:k].tolist())
        mine = set(got.indices[got.indptr[q]:got.indptr[q + 1]].tolist())
        kth = order[k - 1]
        for lab in exact ^ mine:
            assert abs(v_all[q, lab] - v_all[q, kth]) <= e_all[q, lab] + e_all[q, kth], (
                f"{what} {pp}: query {q} label {lab} {'missing from' if lab in exact else 'wrongly in'} the top-{k}")


# ------------------------------------------------------------------------------------------------ runner
def _same_bits(got, want, what):
    assert_csr_parity(got, want, rtol=0.0, what=what)
    assert np.array_equal(np.asarray(got.data, dtype=np.float32).view(np.uint32),
                          np.asarray(want.data, dtype=np.float32).view(np.uint32)), f"{what}: score bits differ"


class _Model(object):
    def __init__(self, clib, have_ref, folder, layers):
        from oracle import ref, restatement
        from pecos_b200.xlinear import XLinearModel

        self.folder, self.layers = folder, layers
        self.m = XLinearModel.load(folder, is_predict_only=True)
        self.c = clib.clib_float32
        self.h = self.m.model.model_chain
        self.depth = len(layers)
        self.oracles = [restatement.OracleXLinear(os.path.join(folder, "ranker"))]
        if have_ref:
            self.oracles.append(ref.RefXLinear(os.path.join(folder, "ranker")))

    def ids(self):
        kid = (c_int * (2 * self.depth))()
        self.c.pb200_xlinear_get_kernel_ids(self.h, kid)
        return [(kid[2 * d], kid[2 * d + 1]) for d in range(self.depth)]

    def cm_info(self, layer):
        """(images built, direct, column cap, virtual chunks, image bytes, warps) chosen at load time; layer -1: prefix"""
        out = (c_uint64 * 6)()
        assert self.c.pb200_xlinear_cm_info(self.h, layer, out) == 0
        return tuple(int(v) for v in out)

    def prefix_used(self):
        prof = (c_double * (2 * self.depth))()
        self.c.pb200_xlinear_get_profile(self.h, prof)
        return prof[1] == 0.0 and prof[2] == 0.0

    def run(self, X, beam, topk, modes, expect, pps=("l3-hinge", "noop"), what="", sub=None, f64=True, profile=False):
        """Predicts X in every kernel mode of `modes` (the first is the baseline) and post-processor of `pps`.  expect(mode,
        pp, ids) asserts on the kernel ids [(score, top-k) per layer] of the call (with profile: (ids, prefix used))."""
        out = {}
        try:
            for pp in pps:
                base = None
                for mode in modes:
                    self.c.pb200_xlinear_set_lookup(self.h, mode)
                    if profile:
                        self.c.pb200_xlinear_set_profile(self.h, 1)
                        self.c.pb200_xlinear_reset_profile(self.h)
                    got = self.m.predict(X, beam_size=beam, only_topk=topk, post_processor=pp)
                    info = self.ids()
                    if profile:
                        info = (info, self.prefix_used())
                        self.c.pb200_xlinear_set_profile(self.h, 0)
                    expect(mode, pp, info)
                    if base is None:
                        base = got
                    else:
                        _same_bits(got, base, f"{what} {pp} mode {mode} vs mode {modes[0]}")
                rows = np.arange(X.shape[0]) if sub is None else sub
                Xs = X[rows]
                for o in self.oracles:
                    assert_csr_parity(base[rows], o.predict(Xs, beam, pp, topk), what=f"{what} {pp} vs {type(o).__name__}")
                if f64:
                    _f64_check(self.layers, 1.0, Xs, base[rows], pp, topk=topk if self.depth == 1 else None, what=what)
                out[pp] = base
        finally:
            self.c.pb200_xlinear_set_lookup(self.h, 1)
        return out


def _expect(table):
    """table: {mode: {layer: (score id or None, top-k id or None)}}"""
    def check(mode, pp, ids):
        for layer, (s, t) in table.get(mode, {}).items():
            if s is not None:
                assert ids[layer][0] == s, f"mode {mode} {pp}: layer {layer} score kernel {ids[layer][0]}, expected {s}"
            if t is not None:
                assert ids[layer][1] == t, f"mode {mode} {pp}: layer {layer} top-k kernel {ids[layer][1]}, expected {t}"
    return check


# ------------------------------------------------------------------------------------------------ query-warp kernel
@pytest.fixture(scope="module")
def qw_model(tmp_path_factory, gpu_clib, have_ref):
    """33 layer-1 chunks of 8 columns over 1,200 features with dense weights (many matched rows per query)."""
    D = 1200
    layers = _two_layer(401, [8] * 33, D, 120)
    folder = _save(str(tmp_path_factory.mktemp("qw")), layers)
    return _Model(gpu_clib, have_ref, folder, layers), D


@pytest.mark.parametrize("beam", [31, 32, 33])
def test_query_warp_beam_slots(qw_model, beam):
    """kQwSlots = 32: the query-warp kernel takes a beam of up to 32 chunks; 33 goes to the feature-map kernel.  Rows of
    300 features against 120-entry columns match hundreds of rows across the beam: several apply passes of 128."""
    mdl, D = qw_model
    X = _queries(411, D, [300] * 20 + [512])
    s = 3 if beam <= 32 else 1
    mdl.run(X, beam, 10, [6, 3, 2], _expect({3: {1: (s, None)}, 2: {1: (1, None)}}), what=f"qw beam {beam}")


@pytest.mark.parametrize("nnz", [512, 513])
def test_query_warp_query_nnz(qw_model, nnz):
    """kQwQCap = 512: the longest row of the batch decides; at 513 the layer goes to the feature-map kernel."""
    mdl, D = qw_model
    X = _queries(412 + nnz, D, [nnz] + [40] * 12)
    s = 3 if nnz <= 512 else 1
    mdl.run(X, 20, 10, [6, 3], _expect({3: {0: (s, None), 1: (s, None)}}), what=f"qw nnz {nnz}")


@pytest.mark.parametrize("width", [2048, 2049])
def test_query_warp_candidate_row_and_block_sort(tmp_path, gpu_clib, have_ref, width):
    """One chunk of 2048 / 2049 columns: kQwNCap = 2048 candidate floats for the query-warp kernel, and kSortCap = 2048
    valid candidates for the block top-k's single sort (2049 streams).  Warp select with k = 64 / 65 (kSelK)."""
    D = 1000
    layers = _flat_layers(421, width, D, 20)
    mdl = _Model(gpu_clib, have_ref, _save(str(tmp_path / "m"), layers), layers)
    X = _queries(422, D, [60] * 16 + [120])
    qw = 3 if width <= 2048 else 1
    mdl.run(X, 0, 10, [6, 3, 0, 4], _expect({3: {0: (qw, 2)}, 0: {0: (0, 0)}, 4: {0: (1, 1)}, 6: {0: (1, 2)}}),
            pps=("l3-hinge", "noop", "log-sigmoid"), what=f"flat {width}")
    for k in (64, 65):
        mdl.run(X, 0, k, [4, 0], _expect({4: {0: (None, 1 if k <= 64 else 0)}, 0: {0: (0, 0)}}),
                pps=("l3-hinge", "log-sigmoid"), what=f"flat {width} k={k}")


# ------------------------------------------------------------------------------------------------ feature-map / row-list / dense
@pytest.fixture(scope="module")
def cover_model(tmp_path_factory, gpu_clib, have_ref):
    """Layer-1 chunks of 128, 129, 64 and 257 columns whose rows are exactly features [0, 600) of 2,000."""
    D, R = 2000, 600
    layers = _two_layer(431, [128, 129, 64, 257], D, 4, cover=R)
    folder = _save(str(tmp_path_factory.mktemp("cover")), layers)
    return _Model(gpu_clib, have_ref, folder, layers), D, R


def test_match_list_flush_points_and_query_staging(cover_model):
    """Rows matching exactly 126 - 129 and 254 - 257 rows of every chunk (+ the bias row): both sides of the row-list
    kernel's flush at kMFlush = 128 and of the lookup kernel's 256-entry list; chunks of 128 / 129 columns (shared-memory vs
    HBM accumulation, kCSmem = 128); rows of 1024 / 1025 features (kQCap: staged in shared memory or read through L1)."""
    mdl, D, R = cover_model
    matches = [126, 127, 128, 129, 254, 255, 256, 257, 300, 300]
    nnz = [m + 40 for m in matches[:-2]] + [1024, 1025]
    X = _queries(441, D, nnz, cover=R, match_list=matches)
    ids = {0: {1: (0, 0)}, 2: {1: (1, 2)}, 6: {1: (1, 2)}, 3: {1: (1, 2)}}
    mdl.run(X, 4, 10, [6, 0, 2, 3], _expect(ids), what="match counts")
    # the same match counts without the 1024 / 1025-feature rows: every row fits the 1024-entry staging area
    X = _queries(443, D, nnz[:8], cover=R, match_list=matches[:8])
    mdl.run(X, 4, 10, [6, 0, 2], _expect(ids), what="match counts, staged")


def test_dense_queries_wide_and_narrow_chunks(cover_model):
    """Dense rows through the dense-query kernel (id 2) over chunks of 128 / 129 / 257 columns."""
    mdl, D, R = cover_model
    X = _queries(442, D, [100, 127, 128, 129, 400], cover=R, match_list=[50, 127, 128, 129, 256])
    Xd = np.asarray(X.toarray(), dtype=np.float32)
    mdl.run(Xd, 4, 10, [6, 1], _expect({1: {1: (2, 2)}, 6: {1: (2, 2)}}), what="dense")


@pytest.fixture(scope="module")
def wide_root_model(tmp_path_factory, gpu_clib, have_ref):
    """Layer 0: one chunk of 129 columns; layer 1: 129 chunks of 3 columns."""
    D = 800
    layers = _two_layer(451, [3] * 129, D, 30)
    folder = _save(str(tmp_path_factory.mktemp("wide_root")), layers)
    return _Model(gpu_clib, have_ref, folder, layers), D


@pytest.mark.parametrize("beam", [10, 11, 20, 21, 64, 65, 128, 129])
def test_beam_slots_per_warp_and_topk_slots(wide_root_model, beam):
    """b_prev 10 / 11 and 20 / 21 (kWarpsMax = 10 slots per round of warps), 128 / 129 (chunk headers cached in shared
    memory), 64 / 65 (kFltSlots and kSelSlots: the filter and the warp select take at most 64 beam slots)."""
    mdl, D = wide_root_model
    X = _queries(452, D, [50] * 24 + [90])
    qw = 3 if 16 <= beam <= 32 else 1  # default selection: query-warp for 16 - 32 slots over <= 256 candidates
    flt = 2 if beam <= 64 else 0
    sel = 1 if beam <= 64 else 0
    ids = {1: {1: (qw, flt)}, 0: {1: (0, 0)}, 2: {1: (1, flt)}, 4: {1: (None, sel)}}
    mdl.run(X, beam, 10, [6, 1, 0, 2, 4], _expect(ids), pps=("l3-hinge", "noop", "log-sigmoid"), what=f"beam {beam}")
    if beam in (10, 11, 128, 129):
        mdl.run(np.asarray(X.toarray(), dtype=np.float32), beam, 10, [6, 1], _expect({1: {1: (2, flt)}}),
                pps=("l3-hinge",), what=f"dense beam {beam}")


# ------------------------------------------------------------------------------------------------ top-k kernels
@pytest.mark.parametrize("width", [4096, 4097, 8064, 8065, 8192, 8193])
def test_filter_and_warp_select_candidate_rows(tmp_path, gpu_clib, have_ref, width):
    """One chunk of `width` columns: kSelKeysMax = 4096 (warp select), kFltKeysMax = 8192 (filter; its key capacity rounds
    up to 128, so 8064 / 8065 too).  l4-hinge takes the filter, l5-hinge does not (its power is not formed exactly)."""
    D = 1000
    layers = _flat_layers(461 + width, width, D, 16)
    mdl = _Model(gpu_clib, have_ref, _save(str(tmp_path / "m"), layers), layers)
    X = _queries(462, D, [60] * 10 + [100])
    flt = 2 if width <= 8192 else 0
    sel = 1 if width <= 4096 else 0

    def expect(mode, pp, ids):
        want = {1: flt if pp != "l5-hinge" else sel, 4: sel, 0: 0}[mode]
        assert ids[0][1] == want, f"width {width} mode {mode} {pp}: top-k kernel {ids[0][1]}, expected {want}"

    mdl.run(X, 0, 10, [1, 4, 0], expect, pps=("l3-hinge", "noop", "log-sigmoid", "l4-hinge", "l5-hinge"),
            what=f"flat {width}")


@pytest.mark.parametrize("k", [300, 512, 513, 1024, 1025])
def test_block_topk_streaming_and_hbm_sort(tmp_path_factory, gpu_clib, have_ref, k):
    """3,000 candidates (> kSortCap = 2048): k <= 1024 streams through shared memory with KP = next_pow2(k) (512 -> 513
    doubles it), k = 1025 sorts the whole row in HBM.  A 100-column model asks for more labels than exist."""
    D = 1000
    for width in (3000, 100):
        layers = _flat_layers(471 + width, width, D, 16)
        mdl = _Model(gpu_clib, have_ref, _save(str(tmp_path_factory.mktemp(f"blk{width}")), layers), layers)
        X = _queries(472, D, [60] * 8 + [100])
        mdl.run(X, 0, k, [1, 0], _expect({1: {0: (None, 0)}, 0: {0: (0, 0)}}), pps=("l3-hinge", "noop", "log-sigmoid"),
                what=f"flat {width} k={k}")


# ------------------------------------------------------------------------------------------------ chunk-major kernel
@pytest.mark.parametrize("D", [16383, 16384])
def test_chunk_major_direct_table_edge(tmp_path, gpu_clib, have_ref, D):
    """W rows = D + 1 = 16384 / 16385 (kCmDirectRows): a direct feature table, or the feature map.  By default (mode 1)
    only direct-table layers take the chunk-major kernel; mode 5 takes it on both.  1,200 queries x 16 beam slots keep the
    pairs above kCmMinPairsPerSm x SMs."""
    layers = _two_layer(481, [8] * 16, D, 40)
    mdl = _Model(gpu_clib, have_ref, _save(str(tmp_path / "m"), layers), layers)
    X = _queries(482, D, [30] * 1200 + [200])
    direct = D + 1 <= 16384

    def expect(mode, pp, ids):
        if mode == 6:
            assert ids[1][0] != 4
        elif mode == 5:
            assert ids[1][0] == 4, f"mode 5: leaf kernel {ids[1][0]}"
        elif mode == 1:
            assert (ids[1][0] == 4) == direct, f"D + 1 = {D + 1}: leaf kernel {ids[1][0]} in mode 1"

    sub = np.r_[0:40, X.shape[0] - 4:X.shape[0]]
    mdl.run(X, 16, 10, [6, 1, 5], expect, what=f"direct edge {D + 1}", sub=sub)


@pytest.mark.parametrize("widest", [256, 257])
def test_chunk_major_virtual_chunks(tmp_path, gpu_clib, have_ref, widest):
    """The widest chunk at 256 columns (one image per chunk) and 257 (col_cap > 256 fails, the cap loop cuts the chunks
    into ranges of at most 224 = 257 * 7 / 8 columns)."""
    D = 500
    layers = _two_layer(491, [widest, 10, 100, 40], D, 12)
    mdl = _Model(gpu_clib, have_ref, _save(str(tmp_path / "m"), layers), layers)
    X = _queries(492, D, [40] * 60 + [120])
    ok, direct, cap, n_vc, _, _ = mdl.cm_info(1)
    assert (ok, direct) == (1, 1)
    assert (cap, n_vc) == ((256, 4) if widest <= 256 else (224, 5)), f"widest {widest}: cap {cap}, {n_vc} virtual chunks"
    mdl.run(X, 4, 10, [6, 5], _expect({5: {1: (4, None)}}), what=f"widest {widest}")


@pytest.mark.parametrize("outside", [False, True])
def test_chunk_major_cap_loop_entry_edge(tmp_path, gpu_clib, have_ref, outside):
    """The cap loop's first step: a widest chunk of 200 columns with exactly the entries an uncut image takes, or one more
    (`_cap_loop_layers` derives the count from cm_shape's layout).  Inside the leaf keeps cap 200 and 9 images; outside it
    is cut at 175 columns into 10.  Both take the chunk-major kernel in mode 5 with the bits of mode 6."""
    layers, e = _cap_loop_layers(outside)
    mdl = _Model(gpu_clib, have_ref, _save(str(tmp_path / "m"), layers), layers)
    ok, direct, cap, n_vc, img, _ = mdl.cm_info(1)
    assert (ok, direct) == (1, 1)
    if outside:
        assert (cap, n_vc) == (175, 10), f"{e} entries: cap {cap}, {n_vc} virtual chunks"
    else:
        assert (cap, n_vc, img) == (200, 9, _cm_direct_image_bytes(CAP_D + 1, e)), f"{e} entries: cap {cap}, {n_vc}, {img} B"
    X = _queries(603, CAP_D, [60] * 40 + [200])
    mdl.run(X, 9, 10, [6, 5], _expect({5: {1: (4, None)}}), what=f"cap loop {e} entries")


@pytest.mark.parametrize("outside", [False, True])
def test_prefix_image_budget_edge(tmp_path, gpu_clib, have_ref, outside):
    """The merged prefix image of 64 columns with exactly the entries that fit next to 4 warps in 224 KB, or one more
    (`_prefix_budget_layers`): the prefix launch runs in mode 5 inside and not outside."""
    layers, e = _prefix_budget_layers(outside)
    mdl = _Model(gpu_clib, have_ref, _save(str(tmp_path / "m"), layers), layers)
    ok, direct, cap, _, img, _ = mdl.cm_info(-1)
    if outside:
        assert ok == 0, f"{e} merged entries: prefix image built"
    else:
        assert (ok, direct, cap, img) == (1, 1, 64, _cm_direct_image_bytes(PFX_D + 1, e))
    X = _queries(612, PFX_D, [40] * 40 + [150])

    def expect(mode, pp, info):
        ids, used = info
        assert used == (mode == 5 and not outside), f"{e} merged entries: prefix {'' if used else 'not '}used in mode {mode}"

    mdl.run(X, 10, 10, [7, 5, 6], expect, what=f"prefix budget {e} entries", profile=True)


def test_chunk_major_no_cap_fits(tmp_path, gpu_clib, have_ref):
    """A chunk with 66,001 rows (every feature of 66,000 plus the bias): r_max >= 65535 fails every cap, so the layer never
    takes the chunk-major kernel, even in mode 5."""
    D, n = 66000, 64
    r = np.arange(D)
    rows = np.concatenate([r, np.full(n, D)])
    cols = np.concatenate([r % n, np.arange(n)])
    vals = np.random.default_rng(501).standard_normal(rows.size).astype(np.float32) * np.float32(0.2)
    W = smat.csc_matrix((vals, (rows, cols)), shape=(D + 1, n))
    W.sort_indices()
    layers = [(W, smat.csc_matrix(np.ones((n, 1), dtype=np.float32)))]
    mdl = _Model(gpu_clib, have_ref, _save(str(tmp_path / "m"), layers), layers)
    X = _queries(502, D, [200] * 20 + [600])
    mdl.run(X, 0, 10, [6, 5], _expect({5: {0: (1, None)}}), what="no cap fits")


@pytest.mark.parametrize("sizes,prefix", [([1, 50], True), ([8, 248], True), ([8, 249], False), ([9, 60], False)])
def test_prefix_limits(tmp_path, gpu_clib, have_ref, sizes, prefix):
    """The prefix launch scores layers 0 and 1 in one pass when layer 0 has at most kCmPrefixTop0 = 8 nodes and the two
    layers at most 256 columns together; 9 nodes, or 8 + 249, score layer by layer.  Mode 5 (any tile size) against mode 7
    (no prefix) and mode 6; the prefix leaves layer 0's top-k and layer 1's score time slots at 0 ms."""
    D = 600
    n0, n1 = sizes
    widths = synth._split_sizes(np.random.default_rng(511), n1, n0, even=True)
    layers = _two_layer(512, list(widths), D, 20)
    mdl = _Model(gpu_clib, have_ref, _save(str(tmp_path / "m"), layers), layers)
    X = _queries(513, D, [40] * 40 + [90])

    def expect(mode, pp, info):
        ids, used = info
        if mode == 5:
            assert used == prefix, f"{sizes}: prefix {'not ' if prefix else ''}used"
            if prefix:
                assert ids[0][0] == 4
        else:
            assert not used, f"{sizes}: prefix used in mode {mode}"

    mdl.run(X, 10, 10, [7, 5, 6], expect, what=f"prefix {sizes}", profile=True)


def test_feature_map_budget_that_drops_only_the_leaf(tmp_path, gpu_clib, have_ref, monkeypatch):
    """PB200_FEATMAP_MB = 1 at load: a layer's map takes n_chunks x ceil(W rows / 32) x 8 bytes, so with W rows = 16,384
    layers 0 - 2 (1 / 8 / 128 chunks: 4 + 32 + 512 KB) keep their maps and the leaf (1,024 chunks: 4 MB) loses its own.
    The chunk-major kernel needs EVERY layer's map, so no layer takes it, not even in mode 5; the prefix launch needs only
    layers 0 and 1 and still serves them (id 4); the leaf streams row lists.  On a full-budget handle the same batch (sub-tiles
    of 6,528 rows, above 48 per SM) runs the prefix and chunk-major kernels everywhere.  Both handles return the same bits
    in every mode."""
    D = 16383
    layers = random_tree(531, [8, 128, 1024, 4096], D, 16)
    folder = _save(str(tmp_path / "m"), layers)
    X = synth.make_queries(532, 26000, D, 40)
    sub = np.r_[0:30, X.shape[0] - 10:X.shape[0]]
    full = _Model(gpu_clib, have_ref, folder, layers)
    monkeypatch.setenv("PB200_FEATMAP_MB", "1")
    part = _Model(gpu_clib, have_ref, folder, layers)
    assert full.c.pb200_xlinear_set_lookup(full.h, 1) == 1
    assert part.c.pb200_xlinear_set_lookup(part.h, 1) == 0, "the leaf must lose its feature map"

    def expect(table):
        def check(mode, pp, info):
            ids, used = info
            want_scores, want_used = table[mode]
            assert [s for s, _ in ids] == want_scores, f"mode {mode} {pp}: score kernels {ids}, expected {want_scores}"
            assert used == want_used, f"mode {mode} {pp}: prefix {'' if used else 'not '}used"
        return check

    want = full.run(X, 10, 10, [1, 0], expect({1: ([4, 4, 4, 4], True), 0: ([0, 0, 0, 0], False)}),
                    what="full feature-map budget", sub=sub, profile=True)
    got = part.run(X, 10, 10, [1, 5, 7, 0],
                   expect({1: ([4, 4, 1, 0], True), 5: ([4, 4, 1, 0], True), 7: ([1, 1, 1, 0], False), 0: ([0, 0, 0, 0], False)}),
                   what="leaf without a feature map", sub=sub, f64=False, profile=True)
    for pp in want:
        _same_bits(got[pp], want[pp], f"{pp}: leaf without a feature map vs the full budget")


# ------------------------------------------------------------------------------------------------ wide beam
def test_wide_beam_runs_at_the_limit_and_raises_past_it(tmp_path, gpu_clib, have_ref):
    """kXlBeamMaxTopk = 15,701: the block top-k's shared memory (2048 keys + 3 words per beam slot <= 200 KB).  A beam of
    15,701 of 16,000 layer-1 nodes runs (about 31,000 candidates per query at the leaf; layer 1 sorts 16,000 in HBM for
    k = 15,701); 15,702 raises ValueError before any GPU work, and the model keeps working.  Modes 1 and 0 (row-list
    scores) agree bit for bit.  The python chain (is_predict_only=False, one single-layer call per layer) raises the same
    ValueError before the leaf's call, and at 15,701 returns the predict-only handle's bits."""
    from pecos_b200.xlinear import XLinearModel

    D = 200
    layers = synth.make_tree_model(521, [16, 16000, 32000], D, 4, bias=1.0)
    layers = [(smat.csc_matrix(W, dtype=np.float32), smat.csc_matrix(C, dtype=np.float32)) for W, C in layers]
    folder = _save(str(tmp_path / "m"), layers)
    mdl = _Model(gpu_clib, have_ref, folder, layers)
    X = _queries(522, D, [20, 30, 25])
    with pytest.raises(ValueError, match="15701"):
        mdl.m.predict(X, beam_size=15702, only_topk=10)
    got = mdl.run(X, 15701, 10, [1, 0], _expect({1: {1: (None, 0), 2: (None, 0)}, 0: {2: (0, 0)}}),
                  pps=("l3-hinge", "noop", "log-sigmoid"), what="beam 15701")
    with pytest.raises(ValueError):
        mdl.m.predict(X, beam_size=20000, only_topk=10)
    mdl.run(X, 20, 10, [1], _expect({}), pps=("l3-hinge",), what="after the refused call")
    chain = XLinearModel.load(folder, is_predict_only=False)
    with pytest.raises(ValueError, match="15702 nodes"):
        chain.predict(X, beam_size=15702, only_topk=10)
    _same_bits(chain.predict(X, beam_size=15701, only_topk=10), got["l3-hinge"], "python chain, beam 15701")
