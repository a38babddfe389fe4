"""GPU tests for the bucketing of chunk-major pairs (xl_cm_count_kernel / xl_cm_scatter_kernel in
pecos_b200/csrc/xlinear_cm_kernel.cuh): each CTA counts its pairs per virtual chunk in a shared-memory histogram of
kCmBinWindow bins, adds each non-empty bin to the bucket counter once, and places its pairs in one reserved run per bucket.
A layer with more virtual chunks than the window takes one pass per window.

Every case goes through `_check` of test_chunk_major_claims_gpu.py: the batch is predicted with its rows shuffled, so a pair
that was never placed (or placed twice over another) leaves a stale or wrong score, and the result must equal kernel mode 6
(no chunk-major kernel) bit for bit, and the oracles."""
from ctypes import c_int

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .test_chunk_major_claims_gpu import _check
from .util import csr_with_empty_rows, random_tree

pytestmark = pytest.mark.gpu

BIN_WINDOW = 8192  # kCmBinWindow


def _kernel_ids(clib, folder, X, depth, mode, beam, topk):
    """Score kernel id per layer of one prediction under kernel `mode` (4 = chunk-major), and the prediction."""
    from pecos_b200.xlinear import XLinearModel

    m = XLinearModel.load(folder, is_predict_only=True)
    c = clib.clib_float32
    h = m.model.model_chain
    kid = (c_int * (2 * depth))()
    c.pb200_xlinear_set_lookup(h, mode)
    try:
        got = m.predict(X, beam_size=beam, only_topk=topk)
        c.pb200_xlinear_get_kernel_ids(h, kid)
    finally:
        c.pb200_xlinear_set_lookup(h, 1)
    return [kid[2 * d] for d in range(depth)], got


@pytest.fixture(scope="module")
def eurlex(tmp_path_factory):
    cfg = synth.WORKLOADS["eurlex-4k"]
    folder, _, _ = synth.build_workload("eurlex-4k", str(tmp_path_factory.mktemp("eurlex") / "m"), scale_queries=8)
    return folder, cfg


def test_eurlex_leaf_and_host_csr_subtiles(eurlex, gpu_clib, have_ref):
    """bench.py's eurlex-4k batch through the host CSR path: four sub-tiles of ~3,860 rows each bucket layer 1 (about
    15,400 pairs on 4 chunks per sub-tile), then the leaf buckets 154,490 pairs on 64 chunks."""
    folder, cfg = eurlex
    X = synth.make_queries(cfg["query_seed"], cfg["Q"], cfg["D"], cfg["nnz_per_row"])
    ids, _ = _kernel_ids(gpu_clib, folder, X, 3, 1, cfg["beam_size"], cfg["only_topk"])
    assert ids[1:] == [4, 4], f"layers 1 and 2 must run the chunk-major kernel, got {ids}"
    _check(gpu_clib, have_ref, folder, X, 3, 1, "eurlex host csr", beam=cfg["beam_size"], topk=cfg["only_topk"], runs=2,
           oracle_rows=np.r_[0:32], pps=("l3-hinge",))


def test_pairs_piled_on_1_4_and_64_chunks(eurlex, gpu_clib, have_ref):
    """Kernel mode 7 (no prefix kernel) on 30,000 eurlex-4k queries: each host sub-tile of 7,500 rows puts every query's
    layer-0 pair on one chunk, its layer-1 pairs on 4 chunks, and the leaf's on 64."""
    folder, cfg = eurlex
    X = synth.make_queries(31, 30000, cfg["D"], cfg["nnz_per_row"])
    ids, _ = _kernel_ids(gpu_clib, folder, X, 3, 7, cfg["beam_size"], cfg["only_topk"])
    assert ids == [4, 4, 4], f"every layer must run the chunk-major kernel, got {ids}"
    _check(gpu_clib, have_ref, folder, X, 3, 7, "piled", beam=cfg["beam_size"], topk=cfg["only_topk"], runs=2,
           oracle_rows=np.r_[0:32], pps=("l3-hinge",))


def _leaf_over_chunks(tmp_path, seed, widths, heavy=()):
    """A 3-layer tree whose leaf has one chunk per entry of `widths` (columns of leaf chunk j = widths[j]); layer-1 nodes in
    `heavy` get a large bias weight, so their leaf chunks are in nearly every beam."""
    D, n1 = 400, len(widths)
    layers = random_tree(seed, [4, n1], D, 24, bias=1.0)
    W1 = smat.lil_matrix(layers[1][0])
    for j in heavy:
        W1[D, j] = 8.0
    layers[1] = (smat.csc_matrix(W1, dtype=np.float32), layers[1][1])
    W_leaf, _ = synth.make_tree_model(seed + 1, [1, int(np.sum(widths))], D, 24, bias=1.0)[1]
    layers.append((smat.csc_matrix(W_leaf, dtype=np.float32), synth._contiguous_codes(widths)))
    folder = str(tmp_path / f"m{seed}")
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=8)
    return folder


@pytest.mark.parametrize("case", ["at_window", "past_window"])
def test_virtual_chunks_at_and_past_the_bin_window(tmp_path, gpu_clib, have_ref, case):
    """Leaf layers (forced onto the chunk-major kernel, mode 5) with exactly BIN_WINDOW virtual chunks (one pass), and with
    two chunks cut into two column ranges (nr = 2) so that BIN_WINDOW + 2 virtual chunks take two passes: chunk 0 shifts the
    others by one, and chunk BIN_WINDOW - 2's ranges are virtual chunks BIN_WINDOW - 1 and BIN_WINDOW, one on each side of
    the window edge.  Both cut chunks are in nearly every beam."""
    rng = np.random.default_rng(851)
    widths = rng.integers(1, 4, BIN_WINDOW)
    heavy = ()
    if case == "past_window":
        heavy = (0, BIN_WINDOW - 2)
        widths[list(heavy)] = 300  # wider than the kernel's 256 columns: cut in two
    folder = _leaf_over_chunks(tmp_path, 852, widths, heavy)
    X = synth.make_queries(853, 3000, 400, 40)
    _check(gpu_clib, have_ref, folder, X, 3, 5, case, runs=2, oracle_rows=np.r_[0:100])


def test_wide_beam(tmp_path, gpu_clib, have_ref):
    """A beam of 600 over 1,024 leaf chunks: each warp walks 19 rounds of 32 beam slots per query, 360,000 pairs."""
    D = 400
    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, random_tree(861, [8, 1024, 6000], D, 24, bias=1.0), bias=1.0, only_topk=8)
    X = synth.make_queries(862, 600, D, 40)
    _check(gpu_clib, have_ref, folder, X, 3, 5, "wide beam", beam=600, runs=2, oracle_rows=np.r_[0:20])


def test_empty_beams(tmp_path, gpu_clib, have_ref):
    """A pruned tree: many layer-0 nodes keep no children, so with a beam of 1 or 2 a query whose best layer-0 nodes are
    childless reaches the leaf with an empty beam (an empty output row); queries without features are in the batch too."""
    D = 400
    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, random_tree(871, [16, 24, 800], D, 24, bias=1.0, prune=0.5), bias=1.0, only_topk=8)
    X = csr_with_empty_rows(synth.make_queries(872, 3000, D, 40), [0, 1, 1500, 2999])
    for beam in (1, 2):
        ids, got = _kernel_ids(gpu_clib, folder, X, 3, 5, beam, 8)
        assert ids[2] == 4, f"beam {beam}: the leaf must run the chunk-major kernel, got {ids}"
        empty = np.diff(got.indptr) == 0
        assert empty.any() and not empty.all(), f"beam {beam}: the batch must mix empty and non-empty beams"
        _check(gpu_clib, have_ref, folder, X, 3, 5, f"empty beams {beam}", beam=beam, runs=2, oracle_rows=np.r_[0:100])


def test_workspace_tiles(tmp_path, gpu_clib, have_ref, monkeypatch):
    """PB200_WORKSPACE_MB=64 cuts 20,000 queries into tiles of ~8,700 rows; each tile buckets its pairs at its workspace
    offset, per layer (mode 7)."""
    D = 400
    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, random_tree(881, [2, 4, 1800], D, 24, bias=1.0), bias=1.0, only_topk=10)
    X = synth.make_queries(882, 20000, D, 24)
    monkeypatch.setenv("PB200_WORKSPACE_MB", "64")
    _check(gpu_clib, have_ref, folder, X, 3, 7, "workspace tiles", runs=2, oracle_rows=np.r_[0:100])
