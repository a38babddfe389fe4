"""GPU tests for the accumulate phase of the chunk-major score kernel (pecos_b200/csrc/xlinear_cm_kernel.cuh), which carries
each lane's hit rows from one round of 8 query features into the next: after round r's lookup the warp runs only the trips
that finish round r - 1's hits, and a lane that finishes early goes on into round r's.  The queries here make that carry
as uneven as possible: a lane's hits cluster in one or two of its rounds (the other features own no weight row), some rows
are longer than a round's trips, feature indices repeat across a round boundary, and rows hold 0, 3, 8 or 9 features.
Every variant of the kernel (direct table with 2 and 4 staging rounds, feature map, the prefix launch) must return the
same bits as the query-major kernels (kernel mode 6) and match the oracles."""
import os
from ctypes import c_double, c_int

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .util import assert_csr_parity, random_tree

pytestmark = pytest.mark.gpu

ROUND = 8  # kCmFeat: query features per round


def _carry_model(seed, sizes, D, nnz_per_col, pad_to=None):
    """A random tree whose even features own no weight row (a query hits only on odd features), with two leaf rows (features
    1 and D - 1) that hold an entry in every column: a lane that hits one adds a whole chunk's width of entries.  pad_to:
    the feature space grows to that many features, the new ones without weights."""
    rng = np.random.default_rng(seed + 1)
    layers = random_tree(seed, sizes, D, nnz_per_col, bias=1.0)
    out = []
    for d, (W, C) in enumerate(layers):
        W = smat.coo_matrix(W)
        keep = (W.row >= D) | (W.row % 2 == 1)
        if d == len(layers) - 1:
            keep &= ~np.isin(W.row, [1, D - 1])
        rows, cols, vals = W.row[keep], W.col[keep], W.data[keep]
        if d == len(layers) - 1:
            rows = np.concatenate([rows, np.repeat([1, D - 1], W.shape[1])])
            cols = np.concatenate([cols, np.tile(np.arange(W.shape[1]), 2)])
            vals = np.concatenate([vals, rng.normal(size=2 * W.shape[1]).astype(np.float32)])
        n_rows = W.shape[0]
        if pad_to is not None:
            rows = np.where(rows >= D, rows + (pad_to - D), rows)  # the bias row stays last
            n_rows += pad_to - D
        Wn = smat.csc_matrix((vals.astype(np.float32), (rows, cols)), shape=(n_rows, W.shape[1]))
        Wn.sum_duplicates()
        Wn.sort_indices()
        out.append((Wn, C))
    return out


def _clustered_queries(seed, n, D, rounds, n_feat=None):
    """n rows of rounds x 8 sorted features each; query q hits (odd features) only in round q % rounds, and every third
    query also in round (q + 2) % rounds; every fifth starts with feature 1 (a row with an entry in every column).  The first
    rows are special: 0, 3, 8 and 9 features, a feature repeated across each round boundary, and feature D - 1 last."""
    rng = np.random.default_rng(seed)
    n_feat = n_feat or D
    half = D // 2
    indptr, indices = [0], []
    for q in range(n):
        nnz = ROUND * rounds
        if q in (0, 1, 2, 3):
            nnz = (0, 3, 8, 9)[q]
        base = np.sort(rng.choice(np.arange(1, half - 1), size=nnz, replace=False))
        hit = np.zeros(nnz, dtype=bool)
        for r in (q % rounds, (q + 2) % rounds if q % 3 == 0 else -1):
            hit[r * ROUND:(r + 1) * ROUND] = r >= 0
        if q < 4:
            hit[:] = True
        f = 2 * base + hit
        if q % 5 == 0 and nnz:
            f[0] = 1
        if q == 4 or q % 7 == 0:  # repeat: the last feature of each round is the first of the next
            for b in range(ROUND, nnz, ROUND):
                f[b] = f[b - 1]
        if q % 11 == 0 and nnz:
            f[-1] = D - 1
        if n_feat > D and q % 2 == 1 and nnz:
            f[-1] = n_feat - 1 - (q % 13)  # a feature without weights beyond the model's own range
        indices += list(np.sort(f))
        indptr.append(len(indices))
    data = rng.uniform(0.1, 1.0, size=len(indices)).astype(np.float32)
    X = smat.csr_matrix((data, np.asarray(indices, np.int64), np.asarray(indptr, np.int64)), shape=(n, n_feat))
    X.has_sorted_indices = True
    return X


def _same_bits(got, want, what):
    assert_csr_parity(got, want, rtol=0.0, what=what)
    assert np.array_equal(np.asarray(got.data, dtype=np.float32).view(np.uint32),
                          np.asarray(want.data, dtype=np.float32).view(np.uint32)), f"{what}: score bits differ"


def _check(clib, have_ref, folder, X, depth, what, expect_prefix=False, beam=10, topk=8):
    from oracle import ref, restatement
    from pecos_b200.xlinear import XLinearModel

    m = XLinearModel.load(folder, is_predict_only=True)
    c = clib.clib_float32
    h = m.model.model_chain
    kid = (c_int * (2 * depth))()
    prof = (c_double * (2 * depth))()
    try:
        for pp in ("l3-hinge", "noop"):
            c.pb200_xlinear_set_lookup(h, 6)
            want = m.predict(X, beam_size=beam, only_topk=topk, post_processor=pp)
            c.pb200_xlinear_get_kernel_ids(h, kid)
            assert 4 not in [kid[2 * d] for d in range(depth)], f"{what}: kernel mode 6 must not use the chunk-major kernel"
            c.pb200_xlinear_set_lookup(h, 5)
            c.pb200_xlinear_set_profile(h, 1)
            c.pb200_xlinear_reset_profile(h)
            got = m.predict(X, beam_size=beam, only_topk=topk, post_processor=pp)
            c.pb200_xlinear_get_profile(h, prof)
            c.pb200_xlinear_set_profile(h, 0)
            c.pb200_xlinear_get_kernel_ids(h, kid)
            assert kid[2 * (depth - 1)] == 4, f"{what}: the leaf must run the chunk-major kernel"
            # the prefix launch leaves layer 0's top-k slot and layer 1's score slot empty
            assert (prof[1] == 0.0 and prof[2] == 0.0) == expect_prefix, f"{what}: prefix {'not ' if expect_prefix else ''}used"
            _same_bits(got, want, f"{what} {pp}")
            sub = np.r_[0:24, X.shape[0] - 40:X.shape[0]]
            oracles = [restatement.OracleXLinear(os.path.join(folder, "ranker"))]
            if have_ref:
                oracles.append(ref.RefXLinear(os.path.join(folder, "ranker")))
            for o in oracles:
                assert_csr_parity(got[sub], o.predict(X[sub], beam, pp, topk), what=f"{what} {pp} vs {type(o).__name__}")
    finally:
        c.pb200_xlinear_set_lookup(h, 1)


def test_carry_direct_wide_chunks_and_prefix(tmp_path, gpu_clib, have_ref):
    """Leaf chunks of ~62 columns (direct table, two staging rounds); layers 0 and 1 (4 + 24 columns) go through the prefix
    launch."""
    D = 400
    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, _carry_model(301, [4, 24, 1500], D, 24), bias=1.0, only_topk=8)
    X = _clustered_queries(302, 2400, D, rounds=6)
    _check(gpu_clib, have_ref, folder, X, 3, "direct, 2 stages", expect_prefix=True)


def test_carry_direct_narrow_chunks_four_stages(tmp_path, gpu_clib, have_ref):
    """Chunks of <= 16 columns take four staging rounds: the leaf (8 columns per chunk) and the prefix (4 + 12 columns)."""
    D = 400
    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, _carry_model(311, [4, 12, 96], D, 24), bias=1.0, only_topk=8)
    X = _clustered_queries(312, 2400, D, rounds=5)
    _check(gpu_clib, have_ref, folder, X, 3, "direct, 4 stages", expect_prefix=True)


@pytest.mark.parametrize("sizes", [[4, 32, 800], [4, 64, 512]])  # leaf chunks of 25 columns (2 stages) and 8 (4 stages)
def test_carry_feature_map(tmp_path, gpu_clib, have_ref, sizes):
    """A feature space wider than kCmDirectRows (16,384) looks features up in the chunk's feature map instead."""
    D, wide = 600, 17000
    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, _carry_model(321, sizes, D, 24, pad_to=wide), bias=1.0, only_topk=8)
    X = _clustered_queries(322, 2400, D, rounds=4, n_feat=wide)
    _check(gpu_clib, have_ref, folder, X, 3, f"feature map {sizes}")
