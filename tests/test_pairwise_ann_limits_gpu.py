"""PairwiseANN search at the edges of its kernels' limits (csrc/pairwise_engine.cu): columns around the 128-position slice of a
distance work item and the 1,024 entries of the select kernel's fast path and shared-memory replay; more pairs than the select
grid covers in one sweep; batches around the 2^25-entry tile and a column longer than a tile; dense widths around the ring
depth switch (10,191 / 10,192) and the widest searchable rows; sparse query rows around the 4,096-entry staging limit and the
8,192-bit filter, base rows around the 64-entry rounds; and NaN / infinite distances.

Every call is checked three ways (_Model.check): against the C restatement (oracle_predict, avx512f order) -- I, M, V and D
bits, two NaNs counting as equal; against oracle/_ref where it is built (bits for sparse models or the avx512f clone, else ids
> 99 % and D within 1e-5); and against a float64 evaluation of every column entry (each finite distance within the float32
accumulation bound, the returned ids the float64 top-k up to near-ties), which catches a mistake the kernel and the
restatement would share.  The counters (pairs, distances, sparse entries, replays -- the last from an exact model of the
fast-path rule) and the launch info (ring depth, per-warp bytes, tiles) are checked on every call.  Every batch holds an empty
column, a column listing one row twice and a query that repeats a base row.
"""
from collections import Counter
from ctypes import POINTER, c_bool, c_float, c_uint32, c_void_p

import numpy as np
import pytest
import scipy.sparse as smat

from tests.test_pairwise_ann_gpu import _pp, _random_case
from tests.util import assert_same_nan

pytestmark = pytest.mark.gpu

SLICE = 128             # column positions per distance work item
SEL_CAP = 1024          # fast path for k up to this; replay in shared memory for n up to this
TILE = 1 << 25          # column entries per tile
SELECT_SLOTS = 132 * 16 * 4  # pairs the select grid covers in one sweep on a 132-SM H100 (sms * 16 CTAs * 4 warps)
WARP_SMEM_MAX = 200 * 1024
FLT_MAX = float(np.finfo(np.float32).max)
EPS32 = 2.0 ** -24
LENS = [0, 1, 127, 128, 129, 255, 256, 257, 1023, 1024, 1025]


# ------------------------------------------------------------------------------------------------------------- helpers
def dense_rule(d):
    """(fits, ring depth, per-warp bytes, row stride) of a dense model of width d, from the row layout of hnsw_host.h."""
    vstride = 64 * ((d // 16 + 3) // 4) + (16 if d % 16 else 0)
    for s in (4, 0):
        per_warp = (vstride * 4 * (1 + s) + 8 * s + SLICE * 4 + 15) & ~15
        if per_warp <= WARP_SMEM_MAX:
            return True, s, per_warp, vstride
    return False, 0, per_warp, vstride


def csc(cols, N, data=None):
    """Y_csc [N x len(cols)] whose column j lists rows cols[j] in that order (duplicates and order kept)."""
    lens = np.array([len(c) for c in cols], np.int64)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = np.concatenate([np.asarray(c, np.int64) for c in cols]) if lens.sum() else np.zeros(0, np.int64)
    if data is None:
        data = ((np.arange(idx.size) % 13) + 1).astype(np.float32) / 4
    Y = smat.csc_matrix((data, idx, indptr), shape=(N, len(cols)))
    Y.has_sorted_indices = False  # stored order is part of the input: never let scipy sort it
    return Y


def with_special_columns(Y, dup_row):
    """Y plus an empty column and a column listing dup_row twice (around two other rows)."""
    cols = [Y.indices[Y.indptr[j]:Y.indptr[j + 1]] for j in range(Y.shape[1])]
    others = [r for r in range(Y.shape[0]) if r != dup_row][:2]
    return csc(cols + [[], [dup_row, others[0], dup_row, others[1]]], Y.shape[0])


def tiles(lens):
    """Tiles the engine forms over a batch of column lengths: consecutive pairs up to TILE entries, or one longer column."""
    t, p = 0, 0
    while p < len(lens):
        t, total, p1 = t + 1, 0, p
        while p1 < len(lens) and not (p1 > p and total + lens[p1] > TILE):
            total += lens[p1]
            p1 += 1
        p = p1
    return t


def _entries(X, Q, q, rows):
    """float64 products of query row q with base rows `rows`: per row (dot, sum |q_i x_i|, products counted, class), class
    0 finite, 1 NaN, 2 +inf (distance -inf), 3 -inf (distance +inf), as float32 products would overflow."""
    if smat.issparse(X):
        Qc = Q[q]
        qv = np.zeros(X.shape[1]); has = np.zeros(X.shape[1], bool)  # noqa: E702
        qv[Qc.indices] = Qc.data; has[Qc.indices] = True  # noqa: E702
        sub = X[rows]
        owner = np.repeat(np.arange(len(rows)), np.diff(sub.indptr))
        hit = has[sub.indices]
        p = sub.data[hit].astype(np.float64) * qv[sub.indices[hit]]
        o = owner[hit]
        n = len(rows)
        dot = np.bincount(o, weights=p, minlength=n).astype(np.float64)  # (integer when no entry matches)
        dot[np.bincount(o, weights=np.isnan(p), minlength=n) > 0] = np.nan
        absum = np.bincount(o, weights=np.where(np.isnan(p), 0, np.abs(p)), minlength=n)
        m = np.bincount(o, minlength=n)
        pos = np.bincount(o, weights=p > FLT_MAX, minlength=n) > 0
        neg = np.bincount(o, weights=p < -FLT_MAX, minlength=n) > 0
    else:
        P = X[rows].astype(np.float64) * np.asarray(Q[q], np.float64)
        dot, absum, m = P.sum(1), np.abs(P).sum(1), np.full(len(rows), X.shape[1])
        pos, neg = (P > FLT_MAX).any(1), (P < -FLT_MAX).any(1)
    cls = np.where(np.isnan(dot) | (pos & neg), 1, np.where(pos, 2, np.where(neg, 3, 0)))
    return dot, absum, m, cls


def f64_check(X, Y, Q, keys, topk, same, out, what=""):
    """Each returned distance against 1 - sum q_i x_i in float64 (finite: within 2 m 2^-24 sum|q_i x_i| + one ulp; else the
    non-finite value the overflowing or NaN products force), and the returned ids against the float64 top-k of the column,
    up to entries within twice that bound of the k-th distance (columns without non-finite distances)."""
    I, M, D, _ = out
    for b, lab in enumerate(keys):
        c0, c1 = int(Y.indptr[lab]), int(Y.indptr[lab + 1])
        n, k = c1 - c0, min(topk, c1 - c0)
        assert (M[b, :k] == 1).all(), what
        if k == 0:
            continue
        rows = np.asarray(Y.indices[c0:c1], np.int64)
        q = 0 if same else b
        parts = [_entries(X, Q, q, rows[s:s + (1 << 20)]) for s in range(0, n, 1 << 20)]
        dot, absum, m, cls = (np.concatenate(a) for a in zip(*parts))
        d64 = 1.0 - dot
        d32 = np.float32(np.clip(np.nan_to_num(d64), -FLT_MAX, FLT_MAX))  # finite entries' final narrowing
        bnd = 2 * m * EPS32 * absum + np.spacing(np.abs(d32)).astype(np.float64)
        order = np.argsort(rows, kind="stable")
        at = order[np.searchsorted(rows[order], I[b, :k].astype(np.int64))]
        assert np.array_equal(rows[at], I[b, :k]), f"returned ids outside the column {what} pair {b}"
        g = D[b, :k].astype(np.float64)
        c = cls[at]
        fin = c == 0
        assert (np.abs(g[fin] - d64[at][fin]) <= bnd[at][fin]).all(), f"distance outside the float32 bound {what} pair {b}"
        assert np.isnan(g[c == 1]).all() and (g[c == 2] == -np.inf).all() and (g[c == 3] == np.inf).all(), \
            f"non-finite distance {what} pair {b}"
        if (cls != 0).any():
            continue
        tol = 2 * bnd.max()
        kth = np.partition(d64, k - 1)[k - 1]
        got = Counter(I[b, :k].tolist())
        for r, cnt in Counter(rows[d64 < kth - tol].tolist()).items():
            assert got[r] >= cnt, f"a float64 top-{k} row is missing {what} pair {b}"
        assert not np.isin(I[b, :k], rows[d64 > kth + tol]).any(), f"a row beyond the float64 top-{k} {what} pair {b}"


def expected_replays(X, Y, Q, keys, topk, same, longest=1 << 20):
    """Pairs the select kernel replays: a NaN in the column, k = min(topk, n) > 1,024, more than one entry at the k-th
    distance, or equal distances among the k smallest (dist + 0.0 folds -0.0 onto +0.0).  The column's float32 distances are
    the restatement's with topk >= n.  Pairs with n > longest are left out (their caller knows their path)."""
    from oracle.pairwise import oracle_predict

    lens = np.diff(Y.indptr)[keys]
    sel = np.flatnonzero((lens > 0) & (lens <= longest))
    total = 0
    b = 0
    while b < sel.size:
        width = int(lens[sel[b]])
        e = b
        while e < sel.size and (e - b + 1) * max(width, int(lens[sel[e]])) <= (1 << 23):
            width = max(width, int(lens[sel[e]]))
            e += 1
        chunk = sel[b:e]
        Qs = Q if same else Q[chunk]
        _, _, Dall, _ = oracle_predict(X, Y, Qs, keys[chunk], width, same)
        for j, p in enumerate(chunk):
            n = int(lens[p])
            k = min(topk, n)
            d = Dall[j, :n] + np.float32(0)
            if np.isnan(d).any() or k > SEL_CAP:
                total += 1
                continue
            s = np.sort(d)
            total += int((s == s[k - 1]).sum() != 1 or (np.diff(s[:k]) == 0).any())
        b = e
    return total


class Model(object):
    """One trained model, searched by the engine, the restatement and (where built) the reference library."""

    def __init__(self, X, Y, have_ref):
        from oracle import restatement
        from oracle.pairwise import RefPairwise
        from pecos_b200.pairwise import PairwiseANN

        self.X, self.Y = X, Y
        self.sparse = smat.issparse(X)
        self.m = PairwiseANN.train(X, Y)
        self.ref = RefPairwise.train(X, Y) if have_ref else None
        self.isa = restatement.host_isa()

    def check(self, Q, keys, topk, same=False, what="", long_replays=None):
        """-> (I, M, D, V), counters, launch info.  long_replays: replays expected among columns longer than 2^20 entries
        (None: no such column in the batch)."""
        from oracle.pairwise import oracle_predict

        X, Y = self.X, self.Y
        keys = np.asarray(keys, np.uint32)
        what = f"{what} topk={topk} same={same}"
        s = self.m.searchers_create(_pp(len(keys), topk))
        got = [a.copy() for a in self.m.predict(Q, keys, s, is_same_input=same)]
        cnt, info = s.counters(), s.launch_info()
        want = oracle_predict(X, Y, Q, keys, topk, same)
        assert_same_nan(got, want, "vs restatement " + what)
        if self.ref is not None:
            r = self.ref.predict(Q, keys, topk, same, threads=8)
            if self.sparse or self.isa == 0:
                assert_same_nan(r, want, "restatement vs reference " + what)
            else:  # the reference ran another SIMD clone: summation order differs in the last bits
                assert np.mean(r[0] == want[0]) > 0.99 and np.allclose(r[2], want[2], rtol=1e-5, atol=1e-6, equal_nan=True), what
        f64_check(X, Y, Q, keys, topk, same, got, what)
        if topk == 0 or len(keys) == 0:
            assert info == {"stages": 0, "warps": 0, "per_warp_bytes": 0, "tiles": 0}, info
            return got, cnt, info
        lens = np.diff(Y.indptr)[keys].astype(np.int64)
        assert cnt["pairs"] == len(keys) and cnt["distances"] == int(lens.sum()), (what, cnt)
        if self.sparse:
            row_nnz = np.diff(X.indptr)
            ent = sum(int(row_nnz[Y.indices[Y.indptr[lab]:Y.indptr[lab + 1]]].sum()) for lab in keys)
            assert cnt["sparse_entries"] == ent, (what, cnt, ent)
        else:
            assert cnt["sparse_entries"] == 0
        assert (long_replays is None) == (lens.max() <= (1 << 20)), "long_replays must be given exactly for long columns"
        assert cnt["replays"] == expected_replays(X, Y, Q, keys, topk, same) + (long_replays or 0), (what, cnt)
        assert info["tiles"] == tiles(lens.tolist()), (what, info)
        if self.sparse:
            assert info["stages"] == 0 and info["per_warp_bytes"] <= WARP_SMEM_MAX, info
        else:
            fits, depth, per_warp, _ = dense_rule(X.shape[1])
            assert fits and (info["stages"], info["per_warp_bytes"]) == (depth, per_warp), (what, info)
        assert info["warps"] >= 1
        return got, cnt, info


def _sparse_rows(rng, n, D, nnz, lo=0.1):
    """n csr rows of D columns, row i with nnz[i] entries (strictly ascending indices), values in [lo, lo + 1)."""
    ptr = np.concatenate([[0], np.cumsum(nnz)])
    idx = np.concatenate([np.sort(rng.choice(D, size=int(k), replace=False)) for k in nnz]) if ptr[-1] else np.zeros(0, int)
    return smat.csr_matrix(((rng.random(int(ptr[-1])) + lo).astype(np.float32), idx, ptr), shape=(n, D))


def _queries_with_base_row(X, Q, row):
    """Q with its last row replaced by base row `row` (a query that repeats a base row)."""
    if smat.issparse(X):
        return smat.vstack([Q[:-1], X[row]]).tocsr()
    Q = Q.copy()
    Q[-1] = X[row]
    return Q


# ------------------------------------------------------------------------------------------------ slices and select cap
def _length_case(rng, sparse, tied):
    """Columns of every length in LENS over N = 3,000 rows, plus the empty and the listed-twice columns; d = 70 dense or a
    96-column csr, small-integer values (every sum exact in float32).  Tie-free: component 0 of row r is r + 1 and the
    queries weigh it by 512, more than the other components can add, so every query's distances to distinct rows differ."""
    N = 3000
    d = 96 if sparse else 70
    if sparse:
        X = _sparse_rows(rng, N, d - 1, rng.integers(25, 40, size=N))
        X.data = rng.integers(1, 3, size=X.nnz).astype(np.float32)
        Q = _sparse_rows(rng, len(LENS) + 2, d - 1, np.full(len(LENS) + 2, 60))
        Q.data = rng.integers(1, 3, size=Q.nnz).astype(np.float32)
        lead_x, lead_q = np.arange(1, N + 1), np.full(Q.shape[0], 512)
        if tied:
            lead_x, lead_q = np.zeros(N), np.zeros(Q.shape[0])
        X = smat.csr_matrix(smat.hstack([smat.csr_matrix(lead_x[:, None]), X]), dtype=np.float32)
        Q = smat.csr_matrix(smat.hstack([smat.csr_matrix(lead_q[:, None]), Q]), dtype=np.float32)
        X.sort_indices(); Q.sort_indices()  # noqa: E702
    else:
        X = rng.integers(-1, 2, size=(N, d)).astype(np.float32)
        Q = rng.integers(-1, 2, size=(len(LENS) + 2, d)).astype(np.float32)
        if not tied:
            X[:, 0], Q[:, 0] = np.arange(1, N + 1), 512
    Y = with_special_columns(csc([rng.choice(N, size=n, replace=False) for n in LENS], N), dup_row=5)
    c = Y.indices[Y.indptr[LENS.index(129)]:Y.indptr[LENS.index(129) + 1]]
    base = int(c.max())  # a query equal to row base >= 1,000 weighs component 0 by base + 1: still tie-free
    assert base >= 1000
    return X, Y, _queries_with_base_row(X, Q, base), np.arange(Y.shape[1], dtype=np.uint32)


@pytest.mark.parametrize("tied", [False, True])
@pytest.mark.parametrize("sparse", [False, True])
def test_column_lengths_around_slices_and_select_capacity(gpu_clib, have_ref, sparse, tied):
    rng = np.random.default_rng(10 + 2 * sparse + tied)
    X, Y, Q, keys = _length_case(rng, sparse, tied)
    mdl = Model(X, Y, have_ref)
    lens = np.diff(Y.indptr)[keys]
    topks = sorted({1, 10, SEL_CAP, SEL_CAP + 1} | {t for n in LENS for t in (n - 1, n, n + 1) if t > 0})
    for topk in topks:
        _, cnt, _ = mdl.check(Q, keys, topk, what=f"sparse={sparse} tied={tied}")
        big = int((np.minimum(topk, lens) > SEL_CAP).sum())
        if not tied:  # only k > 1,024 and the listed-twice column can replay
            assert big <= cnt["replays"] <= big + 1, (topk, cnt)
        elif 10 <= topk <= 1000:  # quantised values tie at the boundary of the long columns, in shared and global memory
            assert cnt["replays"] >= 4, (topk, cnt)
    for same in (False, True):
        mdl.check(Q, keys, 0, same)


# ----------------------------------------------------------------------------------------------- select grid-stride loop
def test_select_grid_stride_over_20000_pairs(gpu_clib, have_ref):
    """20,000 pairs, more than the SELECT_SLOTS warps of the select grid, shuffled over empty, fast-path (continuous rows),
    shared-memory replay (quantised rows, n = 500) and global-memory replay (quantised rows, n = 1,500) columns."""
    rng = np.random.default_rng(20)
    d, half = 16, 4000
    X = np.vstack([rng.standard_normal((half, d)), rng.integers(-1, 2, size=(half, d))]).astype(np.float32)
    cols = [rng.choice(half, size=300, replace=False) for _ in range(8)]           # fast path
    cols += [half + rng.choice(half, size=500, replace=False) for _ in range(8)]   # ties, n <= 1,024
    cols += [half + rng.choice(half, size=1500, replace=False) for _ in range(8)]  # ties, n > 1,024
    Y = with_special_columns(csc(cols, 2 * half), dup_row=7)
    B = 20000
    assert B > SELECT_SLOTS
    keys = rng.permutation(np.arange(B) % Y.shape[1]).astype(np.uint32)
    Q = _queries_with_base_row(X, rng.integers(-1, 2, size=(B, d)).astype(np.float32), half + 3)
    mdl = Model(X, Y, have_ref)
    _, cnt, info = mdl.check(Q, keys, 10, what="grid-stride")
    assert info["tiles"] == 1 and cnt["replays"] > 1000, (cnt, info)


# ------------------------------------------------------------------------------------------------------------------ tiles
def test_batch_of_exactly_one_tile_and_one_entry_more(gpu_clib, have_ref):
    """Columns totalling exactly 2^25 entries run as one tile; one more entry makes a second tile."""
    rng = np.random.default_rng(30)
    N, d, n = 40000, 4, 1 << 15
    X = rng.standard_normal((N, d)).astype(np.float32)
    A = rng.permutation(N)[:n]
    C = np.concatenate([[11], rng.permutation(N)[:n - 2], [11]])  # lists row 11 twice
    Y = csc([A, C, [], [12]], N)
    keys = np.array([0] * 600 + [2] + [0] * 423 + [1], np.uint32)
    assert int(np.diff(Y.indptr)[keys].sum()) == TILE
    Q = _queries_with_base_row(X, rng.standard_normal((len(keys), d)).astype(np.float32), int(A[5]))
    mdl = Model(X, Y, have_ref)
    assert mdl.check(Q, keys, 10, what="2^25")[2]["tiles"] == 1
    Q1 = np.vstack([Q, rng.standard_normal((1, d)).astype(np.float32)])
    assert mdl.check(Q1, np.append(keys, 3).astype(np.uint32), 10, what="2^25 + 1")[2]["tiles"] == 2


@pytest.mark.parametrize("same", [False, True])
def test_long_column_pairs_over_several_tiles(gpu_clib, have_ref, same):
    """About 120 pairs on a 300,000-entry column, interleaved with short and empty columns: >= 2 tiles, later tiles' pairs
    read their own query rows (or row 0 with is_same_input), and replays and entries are summed over the tiles."""
    rng = np.random.default_rng(40 + same)
    N, d = 301000, 3
    # the long column's rows are continuous (fast path), the short column's quantised (ties: replays in every tile)
    X = np.vstack([rng.standard_normal((300000, d)), rng.integers(-1, 2, size=(N - 300000, d))]).astype(np.float32)
    Y = with_special_columns(csc([rng.permutation(300000), 300000 + rng.choice(1000, size=40, replace=False)], N), 9)
    keys = np.array([[0, 1, 2, 0, 3][i % 5] for i in range(300)], np.uint32)
    assert (keys == 0).sum() == 120 and 120 * 300000 > TILE
    Q = _queries_with_base_row(X, rng.integers(-1, 2, size=(len(keys), d)).astype(np.float32), 300001)
    mdl = Model(X, Y, have_ref)
    _, cnt, info = mdl.check(Q, keys, 10, same, what="long column")
    assert info["tiles"] >= 2 and cnt["replays"] > 0, (cnt, info)


@pytest.fixture(scope="module")
def longer_than_a_tile(gpu_clib, have_ref):
    """A column of 2^25 + 1 entries (column 0): row 0 (distance exactly 1.0) everywhere except 12 rows of distinct distances
    below 1.0, at the first and last positions and around slice and tile boundaries; short columns 1-3 of 3, 1 and 5 rows,
    an empty column 4 and column 5 listing row 2 twice.  d = 4."""
    rng = np.random.default_rng(50)
    d, n = 4, TILE + 1
    X = np.vstack([np.zeros((1, d)), np.abs(rng.standard_normal((12, d))) + 0.1, rng.standard_normal((20, d))]).astype(np.float32)
    big = np.zeros(n, np.int64)
    at = [0, SLICE - 1, SLICE, SLICE + 1, 2 * SLICE, n // 2, n - SLICE - 1, n - SLICE, TILE - 1, TILE, 1000, 5000]
    big[at] = np.arange(1, 13)
    Y = csc([big, [13, 14, 15], [16], [17, 18, 19, 20, 21], [], [2, 22, 2]], X.shape[0])
    return Model(X, Y, have_ref)


def test_column_longer_than_a_tile_takes_the_fast_path(longer_than_a_tile):
    """short pair, the 2^25 + 1 column, short pair: three tiles; the long column's 10 smallest are distinct, so it is selected
    by the fast path (a lane-0 replay over 2^25 entries in global memory would take minutes)."""
    mdl = longer_than_a_tile
    Q = np.ones((5, 4), np.float32)
    Q[2] = mdl.X[13]
    for topk in (1, 10):
        _, cnt, info = mdl.check(Q, [1, 0, 3, 4, 5], topk, what="2^25 + 1", long_replays=0)
        assert info["tiles"] == 3 and cnt["distances"] == TILE + 1 + 3 + 5 + 3, (cnt, info)


def test_caller_slots_past_each_column_keep_their_values(longer_than_a_tile):
    """Through the C ABI with sentinel-filled I / M / D / V (the Python layer zeroes them first, which would hide a write):
    slot k >= min(topk, n) of every pair keeps its sentinel, over a batch of three tiles."""
    from pecos_b200.core import ScipyDrmF32
    from oracle.pairwise import oracle_predict

    mdl = longer_than_a_tile
    m = mdl.m
    keys = np.array([1, 2, 0, 5, 4, 3], np.uint32)
    topk, B = 8, len(keys)
    Q = np.ones((B, 4), np.float32)
    Q[0] = mdl.X[14]
    sent = [np.full(B * topk, 0xA5A5A5A5, np.uint32), np.full(B * topk, 7, np.uint32),
            np.full(B * topk, -123.5, np.float32), np.full(B * topk, 99.25, np.float32)]
    tok = m.fn_dict["searchers_create"](m.model_ptr, 1)
    try:
        m.fn_dict["predict"](c_void_p(tok), B, topk, ScipyDrmF32.init_from(Q), keys.ctypes.data_as(POINTER(c_uint32)),
                             sent[0].ctypes.data_as(POINTER(c_uint32)), sent[1].ctypes.data_as(POINTER(c_uint32)),
                             sent[2].ctypes.data_as(POINTER(c_float)), sent[3].ctypes.data_as(POINTER(c_float)), c_bool(False))
        from pecos_b200.core import get_clib
        assert get_clib().pairwise_ann_launch_info(c_void_p(tok))["tiles"] == 3
    finally:
        m.fn_dict["searchers_destruct"](c_void_p(tok))
    got = [a.reshape(B, topk) for a in sent]
    want = oracle_predict(mdl.X, mdl.Y, Q, keys, topk)
    lens = np.diff(mdl.Y.indptr)[keys]
    for b in range(B):
        k = min(topk, int(lens[b]))
        assert_same_nan([g[b, :k] for g in got], [w[b, :k] for w in want], f"pair {b}")
        for g, s in zip(got, (0xA5A5A5A5, 7, -123.5, 99.25)):
            assert (g[b, k:] == s).all(), f"pair {b}: a slot past min(topk, n) = {k} was written"
    assert (lens < topk).sum() >= 4


# ----------------------------------------------------------------------------------------------------------- dense widths
WIDTHS = [1, 3, 4, 15, 16, 17, 63, 64, 65, 1024, 4097, 10191, 10192, 51024, 51072]


@pytest.mark.parametrize("d", WIDTHS)
def test_dense_widths_and_ring_depth(gpu_clib, have_ref, d):
    """Ring depth 4 up to d = 10,191, direct loads from 10,192 to the widest searchable rows."""
    rng = np.random.default_rng(d)
    N = 300 if d > 4096 else 2000
    X, Y = _random_case(rng, False, N, 6, d, 0, long_col=250)
    Y = with_special_columns(Y, dup_row=3)
    keys = np.arange(Y.shape[1], dtype=np.uint32)
    Q = _queries_with_base_row(X, rng.standard_normal((len(keys), d)).astype(np.float32), 4)
    mdl = Model(X, Y, have_ref)
    fits, plan = gpu_clib.pairwise_ann_dense_fits(d)
    assert fits and (plan["stages"] == 4) == (d <= 10191)
    for topk in (1, 10, 300):
        info = mdl.check(Q, keys, topk, what=f"d={d}")[2]
        assert (info["stages"], info["per_warp_bytes"]) == (plan["stages"], plan["per_warp_bytes"]), (d, info, plan)


@pytest.mark.parametrize("d", [51025, 51071, 51073])
def test_too_wide_dense_model_raises_before_native_call(gpu_clib, tmp_path, d):
    """Training and saving are allowed; creating searchers and predicting raise ValueError, the searcher's slots untouched."""
    from pecos_b200.pairwise import PairwiseANN

    X = np.ones((3, d), np.float32)
    m = PairwiseANN.train(X, smat.eye(3, 2, dtype=np.float32, format="csc"))
    m.save(str(tmp_path / "wide"))
    assert PairwiseANN.load(str(tmp_path / "wide")).feat_dim == d
    with pytest.raises(ValueError, match="51,072"):
        m.searchers_create(_pp(2, 2))
    s = PairwiseANN.Searchers(m, _pp(2, 2))  # a real token: the native searchers_create does not search
    s.Imat[:] = 77
    s.Dmat[:] = 5.0
    with pytest.raises(ValueError, match="51,024"):
        m.predict(X[:2], np.array([0, 1], np.uint32), s)
    assert (s.Imat == 77).all() and (s.Dmat == 5.0).all()


# --------------------------------------------------------------------------------------------------------- sparse staging
def test_sparse_query_staging_and_base_row_rounds(gpu_clib, have_ref):
    """Query rows of 0, 4,096 (staged), 4,097 and 20,000 entries (read from global memory; the last sets every filter bit)
    against base rows of 0, 1, 63, 64, 65 and 2,000 entries (64-entry rounds), with and without is_same_input."""
    rng = np.random.default_rng(60)
    D, N = 30000, 1200
    nnz = np.concatenate([[0, 1, 63, 64, 65, 2000] * 4, rng.integers(1, 120, size=N - 24)])
    X = _sparse_rows(rng, N, D, nnz)
    Y = with_special_columns(csc([np.arange(24), rng.choice(N, size=300, replace=False), np.arange(24)[::-1],
                                  rng.choice(N, size=SLICE + 1, replace=False)], N), dup_row=4)
    rows = []
    for k in (0, 4096, 4097, 20000):
        c = np.arange(k) if k == 20000 else np.sort(rng.choice(D, size=k, replace=False))
        rows.append(smat.csr_matrix(((rng.random(k) + 0.1).astype(np.float32), c, [0, k]), shape=(1, D)))
    h = ((np.arange(20000, dtype=np.uint64) * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(19)
    assert np.unique(h).size == 8192  # the filter hash of csrc/hnsw_device.cuh (sp_hash): every bit set
    keys = np.arange(Y.shape[1], dtype=np.uint32)
    B = 4 * len(keys)
    Q = _queries_with_base_row(X, smat.vstack([rows[i // len(keys)] for i in range(B)]).tocsr(), 3)
    keys = np.tile(keys, 4)
    assert sorted(set(np.diff(Q.indptr))) == sorted({0, 4096, 4097, 20000, int(np.diff(X.indptr)[3])})
    mdl = Model(X, Y, have_ref)
    for topk in (1, 10, 300):
        mdl.check(Q, keys, topk, what="csr staging")
    mdl.check(rows[2], keys[:len(keys) * 2], 10, same=True, what="csr staging, same 4,097-entry query")


# ---------------------------------------------------------------------------------------------------- non-finite distances
def nonfinite_case(rng, sparse):
    """Rows whose distance to every query is NaN (a NaN component met by the query; products overflowing to +inf and -inf),
    -inf (an overflowing positive product) or +inf (negative), several of each (ties at +-inf), at slice boundaries and
    elsewhere in columns of 40, 300 and 1,100 entries, among finite rows whose products stay small.  Queries put 1e20 on
    components 0 and 1, so |q_i x_i| > FLT_MAX on its own for x_i = +-1e20 and every summation order agrees."""
    N, d = 2000, (200 if sparse else 70)
    if sparse:
        X = _sparse_rows(rng, N, d, rng.integers(5, 30, size=N)).tolil()
        X[:, :2] = 0
        Q = _sparse_rows(rng, 8, d, np.full(8, 60)).tolil()
        Q[:, 0] = 1e20
        Q[:, 1] = 1e20
    else:
        X = rng.standard_normal((N, d)).astype(np.float32)
        X[:, :2] = 0
        Q = rng.standard_normal((8, d)).astype(np.float32)
        Q[:, :2] = 1e20
    kinds = {"nan": range(10, 20), "both": range(20, 30), "pos": range(30, 40), "neg": range(40, 50)}
    for r in kinds["nan"]:
        if sparse:  # a NaN where the query has no entry changes nothing: give the query one there too
            X[r, 2] = np.nan
            Q[:, 2] = 0.5
        else:
            X[r, 5 + r % 50] = np.nan
    for r in kinds["both"]:
        X[r, 0], X[r, 1] = 1e20, -1e20
    for r in kinds["pos"]:
        X[r, 0] = 1e20
    for r in kinds["neg"]:
        X[r, 1] = -1e20
    if sparse:
        X, Q = smat.csr_matrix(X, dtype=np.float32), smat.csr_matrix(Q, dtype=np.float32)
        X.sort_indices(); Q.sort_indices()  # noqa: E702
    # (length, positions, special rows): NaNs alone (no ties, so only the NaN check keeps these off the fast path); every
    # kind with two rows of each infinite kind (ties at -inf and +inf); NaNs with one -inf and one +inf; one NaN at a slice
    # boundary
    layout = ((40, [0, 3, 17], [10, 11, 20]),
              (300, [0, 126, 127, 128, 129, 255, 256, 299], [10, 20, 30, 31, 40, 41] + list(range(12, 19)) + [32, 42, 21]),
              (1100, [127, 128, 1023, 1024], [12, 21, 30, 40]),
              (129, [128], [13]))
    cols = []
    for n, at, pick in layout:
        c = rng.choice(np.arange(100, N), size=n, replace=False)
        rest = np.setdiff1d(np.arange(n), at)
        pos = np.concatenate([at, rng.choice(rest, size=len(pick) - len(at), replace=False)])
        c[pos] = rng.permutation(pick)
        cols.append(c)
    Y = with_special_columns(csc(cols, N), dup_row=20)
    keys = np.arange(Y.shape[1], dtype=np.uint32)
    Qb = Q[np.arange(len(keys)) % Q.shape[0]]
    return X, Y, _queries_with_base_row(X, Qb, 15), keys


@pytest.mark.parametrize("sparse", [False, True])
def test_nan_and_infinite_distances(gpu_clib, have_ref, sparse):
    """Columns with NaN, +inf and -inf distances, topk from 1 past n: the engine replays every pair whose column holds a NaN
    and so places the NaNs where the reference's heap sequence does."""
    rng = np.random.default_rng(70 + sparse)
    X, Y, Q, keys = nonfinite_case(rng, sparse)
    mdl = Model(X, Y, have_ref)
    lens = np.diff(Y.indptr)[keys]
    seen = set()
    for topk in list(range(1, 302)) + [1023, 1024, 1025, 1100, 1101]:
        got, cnt, _ = mdl.check(Q, keys, topk, what=f"non-finite sparse={sparse}")
        D = got[2]
        seen |= {"nan"} if np.isnan(D).any() else set()
        seen |= {"+inf"} if (D == np.inf).any() else set()
        seen |= {"-inf"} if (D == -np.inf).any() else set()
        assert cnt["replays"] >= 4  # the first four columns hold NaNs
    assert seen == {"nan", "+inf", "-inf"}
