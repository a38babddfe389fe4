"""GPU tests for the chunk-major score kernel at the shapes the other chunk-major tests do not reach: the real eurlex-4k leaf
(5,000 features, 46 - 84-column chunks, a 120 KB+ image that leaves fewer than 16 warps per CTA), a layer whose chunk
widths differ by more than 10x (the work-weighted split of the pair list meets empty and very heavy buckets), and a model
whose W repeats a row inside a column (non-canonical W: a chunk row holds the same column twice).  Each must return the
same bits as the query-major kernels (kernel mode 6)."""
import os
from ctypes import c_int

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .util import assert_csr_parity, random_tree

pytestmark = pytest.mark.gpu


def _kernel_ids(c, h, depth):
    kid = (c_int * (2 * depth))()
    c.pb200_xlinear_get_kernel_ids(h, kid)
    return [kid[2 * d] for d in range(depth)]


def _chunk_major_equals_query_major(clib, folder, X, depth, mode, beam=10, topk=10, what=""):
    from pecos_b200.xlinear import XLinearModel

    m = XLinearModel.load(folder, is_predict_only=True)
    c = clib.clib_float32
    h = m.model.model_chain
    try:
        for pp in ("l3-hinge", "noop"):
            c.pb200_xlinear_set_lookup(h, 6)
            want = m.predict(X, beam_size=beam, only_topk=topk, post_processor=pp)
            assert 4 not in _kernel_ids(c, h, depth)
            c.pb200_xlinear_set_lookup(h, mode)
            got = m.predict(X, beam_size=beam, only_topk=topk, post_processor=pp)
            assert _kernel_ids(c, h, depth)[depth - 1] == 4, f"{what}: the leaf must run the chunk-major kernel"
            assert_csr_parity(got, want, rtol=0.0, what=f"{what} {pp}")
            assert np.array_equal(got.data.view(np.uint32), want.data.view(np.uint32)), f"{what} {pp}: score bits differ"
    finally:
        c.pb200_xlinear_set_lookup(h, 1)


def test_eurlex_leaf_shape_default_mode(tmp_path, gpu_clib):
    """The eurlex-4k model of bench.py (same seeds) with 4,000 of its queries: the default mode (1) picks the chunk-major
    kernel for the leaf on its own heuristics."""
    cfg = synth.WORKLOADS["eurlex-4k"]
    folder, _, _ = synth.build_workload("eurlex-4k", str(tmp_path / "m"), scale_queries=8)
    X = synth.make_queries(cfg["query_seed"], 4000, cfg["D"], cfg["nnz_per_row"])
    _chunk_major_equals_query_major(gpu_clib, folder, X, len(cfg["layer_sizes"]), 1, cfg["beam_size"], cfg["only_topk"], "eurlex-4k leaf")


def test_uneven_chunk_widths(tmp_path, gpu_clib):
    """Leaf chunks of 2 - 150 columns (> 10x apart); a fifth of the parents is unreachable, so their buckets are empty."""
    D = 400
    layers = random_tree(731, [4, 32], D, 24, prune=0.2)
    rng = np.random.default_rng(732)
    widths = np.where(np.arange(32) % 4 == 0, rng.integers(100, 151, 32), rng.integers(2, 12, 32))
    n_leaf = int(widths.sum())
    W_leaf, _ = synth.make_tree_model(733, [1, n_leaf], D, 24, bias=1.0)[1]
    layers.append((smat.csc_matrix(W_leaf, dtype=np.float32), synth._contiguous_codes(widths)))
    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=10)
    X = synth.make_queries(734, 3000, D, 40)
    _chunk_major_equals_query_major(gpu_clib, folder, X, 3, 5, what="uneven chunk widths")


def test_repeated_row_inside_a_column(tmp_path, gpu_clib):
    """W of the leaf repeats a row inside some columns (stored twice, different weights): every addition still lands in
    feature order, duplicates in stored order."""
    D = 400
    layers = random_tree(741, [4, 32, 1200], D, 24, bias=1.0)
    W = smat.csc_matrix(layers[-1][0])
    W.sort_indices()
    rng = np.random.default_rng(742)
    indptr, indices, data = [0], [], []
    for j in range(W.shape[1]):
        s, e = W.indptr[j], W.indptr[j + 1]
        rows, vals = list(W.indices[s:e]), list(W.data[s:e])
        if j % 3 == 0 and rows:
            for k in sorted(rng.choice(len(rows), size=min(3, len(rows)), replace=False), reverse=True):
                rows.insert(k + 1, rows[k])
                vals.insert(k + 1, np.float32(rng.normal()))
        indices += rows
        data += vals
        indptr.append(len(indices))
    Wd = smat.csc_matrix((np.asarray(data, np.float32), np.asarray(indices, np.int32), np.asarray(indptr, np.int64)), shape=W.shape)
    assert Wd.nnz > W.nnz and not Wd.has_canonical_format
    layers[-1] = (Wd, layers[-1][1])
    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=10)
    stored = smat.load_npz(os.path.join(folder, "ranker", "2.model", "W.npz"))
    assert stored.nnz == Wd.nnz, "the writer must keep the repeated rows"
    X = synth.make_queries(743, 3000, D, 48)
    _chunk_major_equals_query_major(gpu_clib, folder, X, 3, 5, what="repeated rows")
