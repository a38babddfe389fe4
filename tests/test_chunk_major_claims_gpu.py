"""GPU tests for the run-time schedule of the chunk-major score kernel (pecos_b200/csrc/xlinear_cm_kernel.cuh): its CTAs claim
32-pair slices of a chunk from a per-chunk cursor and move to the chunk with the most unclaimed work when theirs runs dry,
so which CTA scores which pair changes from run to run.  The results must not: every case requires the same ids, counts
and score bits as the query-major kernels (kernel mode 6), run after run, and matches the oracles.  The shapes make CTAs
migrate: one chunk holding most of the work next to many tiny chunks and empty buckets, fewer slices than CTAs, and chunks
cut into column ranges (several virtual chunks per chunk).

The engine's candidate workspace is not cleared between calls, so a pair that no CTA scores would keep whatever the
previous call left at its place.  Every chunk-major run therefore predicts the batch with its rows shuffled (no query on
the workspace row it held in the previous call) and un-shuffles the result: a dropped pair shows another query's scores."""
import os
from ctypes import c_int

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .util import assert_csr_parity, random_tree

pytestmark = pytest.mark.gpu


def _same_bits(got, want, what):
    assert_csr_parity(got, want, rtol=0.0, what=what)
    assert np.array_equal(np.asarray(got.data, dtype=np.float32).view(np.uint32),
                          np.asarray(want.data, dtype=np.float32).view(np.uint32)), f"{what}: score bits differ"


def _moved(rng, prev):
    """A random row order that puts no query on the row `prev` gave it."""
    perm = rng.permutation(prev.size)
    same = np.nonzero(perm == prev)[0]
    if same.size > 1:
        perm[same] = np.roll(perm[same], 1)
    elif same.size == 1:
        i, j = same[0], (same[0] + 1) % prev.size
        perm[i], perm[j] = perm[j], perm[i]
    assert not np.any(perm == prev)
    return perm


def _check(clib, have_ref, folder, X, depth, mode, what, beam=10, topk=8, runs=2, oracle_rows=None,
           pps=("l3-hinge", "noop")):
    """`runs` predictions under kernel `mode`, each of a differently shuffled batch, must all equal kernel mode 6 bit for
    bit once un-shuffled, with the leaf on the chunk-major kernel; oracle_rows (default: all) are also checked against the
    oracles."""
    from oracle import ref, restatement
    from pecos_b200.xlinear import XLinearModel

    m = XLinearModel.load(folder, is_predict_only=True)
    c = clib.clib_float32
    h = m.model.model_chain
    kid = (c_int * (2 * depth))()
    rng = np.random.default_rng(X.shape[0])
    try:
        for pp in pps:
            c.pb200_xlinear_set_lookup(h, 6)
            want = m.predict(X, beam_size=beam, only_topk=topk, post_processor=pp)
            c.pb200_xlinear_get_kernel_ids(h, kid)
            assert 4 not in [kid[2 * d] for d in range(depth)], f"{what}: kernel mode 6 must not use the chunk-major kernel"
            c.pb200_xlinear_set_lookup(h, mode)
            order = np.arange(X.shape[0])  # the rows of the mode-6 call
            for r in range(runs):
                order = _moved(rng, order)
                got = m.predict(X[order], beam_size=beam, only_topk=topk, post_processor=pp)[np.argsort(order)]
                c.pb200_xlinear_get_kernel_ids(h, kid)
                assert kid[2 * (depth - 1)] == 4, f"{what}: the leaf must run the chunk-major kernel"
                _same_bits(got, want, f"{what} {pp} run {r}")
            sub = np.arange(X.shape[0]) if oracle_rows is None else oracle_rows
            oracles = [restatement.OracleXLinear(os.path.join(folder, "ranker"))]
            if have_ref:
                oracles.append(ref.RefXLinear(os.path.join(folder, "ranker")))
            for o in oracles:
                assert_csr_parity(got[sub], o.predict(X[sub], beam, pp, topk), what=f"{what} {pp} vs {type(o).__name__}")
    finally:
        c.pb200_xlinear_set_lookup(h, 1)


def test_eurlex_leaf_same_bits_run_after_run(tmp_path, gpu_clib, have_ref):
    """bench.py's eurlex-4k model and query batch in the default mode, predicted five times: the schedule differs between
    runs, the bits must not."""
    cfg = synth.WORKLOADS["eurlex-4k"]
    folder, _, _ = synth.build_workload("eurlex-4k", str(tmp_path / "m"), scale_queries=8)
    X = synth.make_queries(cfg["query_seed"], cfg["Q"], cfg["D"], cfg["nnz_per_row"])
    _check(gpu_clib, have_ref, folder, X, len(cfg["layer_sizes"]), 1, "eurlex-4k leaf", beam=cfg["beam_size"],
           topk=cfg["only_topk"], runs=5, oracle_rows=np.r_[0:32, X.shape[0] - 32:X.shape[0]], pps=("l3-hinge",))


def test_one_heavy_chunk_many_tiny_and_empty(tmp_path, gpu_clib, have_ref):
    """Layer 1's node 0 owns a 200-column leaf chunk, and a large bias weight on it and on its layer-0 parent puts it into
    nearly every beam; the other leaf chunks have 1 - 6 columns, and a quarter of layer 1 gets a large negative bias
    weight, so their buckets are (nearly always) empty.  With a beam of 2, the heavy chunk gets close to half the pairs and
    most of the work: most CTAs start on it, find it dry after a slice or none, and move on to tiny chunks."""
    D, n1 = 400, 128
    layers = random_tree(811, [4, n1], D, 24, bias=1.0)
    W0 = smat.lil_matrix(layers[0][0])
    W0[D, smat.csr_matrix(layers[1][1])[0].indices[0]] = 8.0  # node 0's parent
    layers[0] = (smat.csc_matrix(W0, dtype=np.float32), layers[0][1])
    W1 = smat.lil_matrix(layers[1][0])
    W1[D, 0] = 8.0
    for j in range(3 * n1 // 4, n1):
        W1[D, j] = -8.0
    layers[1] = (smat.csc_matrix(W1, dtype=np.float32), layers[1][1])
    rng = np.random.default_rng(812)
    widths = np.r_[200, rng.integers(1, 7, n1 - 1)]
    W_leaf, _ = synth.make_tree_model(813, [1, int(widths.sum())], D, 24, bias=1.0)[1]
    layers.append((smat.csc_matrix(W_leaf, dtype=np.float32), synth._contiguous_codes(widths)))
    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=8)
    X = synth.make_queries(814, 3000, D, 40)
    _check(gpu_clib, have_ref, folder, X, 3, 5, "one heavy chunk", beam=2, runs=3, oracle_rows=np.r_[0:200])


def test_fewer_slices_than_ctas(tmp_path, gpu_clib, have_ref):
    """60 queries x a beam of 10 over 32 leaf chunks, forced onto the chunk-major kernel (mode 5): about one slice per
    chunk, far fewer slices than CTAs."""
    D = 400
    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, random_tree(821, [4, 32, 800], D, 24, bias=1.0), bias=1.0, only_topk=8)
    X = synth.make_queries(822, 60, D, 48)
    _check(gpu_clib, have_ref, folder, X, 3, 5, "fewer slices than CTAs", runs=3)


def test_column_range_virtual_chunks(tmp_path, gpu_clib, have_ref):
    """Leaf chunks of ~450 columns (wider than the kernel's 256) are cut into column ranges, each a virtual chunk with its
    own image and claim cursor; a pair is scored once per range."""
    D = 400
    folder = str(tmp_path / "m")
    layers = random_tree(831, [2, 4, 1800], D, 24, bias=1.0)
    # no leaf chunk fits the kernel uncut, so a leaf that runs the chunk-major kernel (checked in _check) runs cut
    assert np.asarray(layers[-1][1].sum(axis=0)).min() > 256
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=8)
    X = synth.make_queries(832, 3000, D, 48)
    _check(gpu_clib, have_ref, folder, X, 3, 5, "column ranges", runs=3, oracle_rows=np.r_[0:200])
