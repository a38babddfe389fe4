"""GPU parity tests for the XR-Linear hot path: CUDA engine (through the C ABI / Python mirror) vs the CPU oracles.

Oracle = oracle/_ref (the reference's own libpecos.cpp, compiled unmodified) when it is present, and always our
plain-C restatement (oracle/liboracle.so).  Bar (BASELINE.json north_star): bit-exact top-k label ids and ranks,
scores within 1e-5 relative.

Mirrors the reference's own test strategy for this path (test/pecos/xmc/xlinear/test_xlinear.py):
  * cross-format / post-processor / batch-vs-realtime consistency ... :106-245
  * mmap vs npz ................................................... :1140-1168
  * pruned trees (set_output_constraint) ........................... :917-1012
"""
import os

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .util import assert_csr_parity, csr_with_empty_rows, random_tree

pytestmark = pytest.mark.gpu

POST_PROCESSORS = ["noop", "sigmoid", "log-sigmoid", "l1-hinge", "l2-hinge", "l3-hinge", "l4-hinge",
                   "log-l1-hinge", "log-l2-hinge", "log-l3-hinge", "log-l4-hinge", "l5-hinge"]


def _oracles(folder, have_ref):
    from oracle import ref, restatement

    out = {"restatement": restatement.OracleXLinear(os.path.join(folder, "ranker"))}
    if have_ref:
        out["reference"] = ref.RefXLinear(os.path.join(folder, "ranker"))
    return out


def _load(folder, **kw):
    from pecos_b200.xlinear import XLinearModel

    return XLinearModel.load(folder, is_predict_only=True, **kw)


def _check(model, oracles, X, what, **kw):
    got = model.predict(X, **kw)
    for name, o in oracles.items():
        want = o.predict(X, kw.get("beam_size", 0), kw.get("post_processor"), kw.get("only_topk", 0))
        assert_csr_parity(got, want, what=f"{what} vs {name} {kw}")
    return got


@pytest.fixture(scope="module")
def small_model(tmp_path_factory, gpu_clib, have_ref):
    folder = str(tmp_path_factory.mktemp("xl_small"))
    layers = random_tree(11, [4, 24, 300], 500, 30, bias=1.0)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=7, post_processor="l3-hinge")
    X = synth.make_queries(12, 97, 500, 40)
    return folder, X, _load(folder), _oracles(folder, have_ref)


def test_attrs_and_layer_type(small_model, gpu_clib):
    folder, X, m, oracles = small_model
    assert (m.depth, m.nr_features, m.nr_labels, m.nr_codes) == (3, 500, 300, 24)
    for name, tid in [("CSC", 0), ("HASH_CHUNKED", 1), ("BINARY_SEARCH_CHUNKED", 2)]:
        mm = _load(folder, weight_matrix_type=name)
        assert mm.model.weight_matrix_type == tid  # the requested type is reported back (pecos/xmc/base.py:1736-1743)
        _check(mm, oracles, X, f"weight_matrix_type={name}", beam_size=5, only_topk=5)


@pytest.mark.parametrize("pp", POST_PROCESSORS)
def test_post_processors_sparse_and_dense(small_model, pp):
    folder, X, m, oracles = small_model
    _check(m, oracles, X, "csr", post_processor=pp, beam_size=4, only_topk=6)
    _check(m, oracles, X[:23].toarray(), "drm", post_processor=pp, beam_size=4, only_topk=6)


@pytest.mark.parametrize("beam,topk", [(1, 1), (2, 10), (10, 10), (20, 20), (3, 1000), (50, 7)])
def test_beam_and_topk(small_model, beam, topk):
    folder, X, m, oracles = small_model
    got = _check(m, oracles, X, "csr", beam_size=beam, only_topk=topk)
    # rows shorter than k are kept whole (inference.hpp:1237)
    assert got.getnnz(axis=1).max() <= topk


def test_default_params_and_kwargs_override(small_model):
    folder, X, m, oracles = small_model
    _check(m, oracles, X, "defaults")  # stored only_topk / post-processor of every layer
    got = m.predict(X, only_topk=3)
    assert (got.getnnz(axis=1) == 3).all()


def test_realtime_single_queries(small_model):
    folder, X, m, oracles = small_model
    for i in [0, 5, 96]:
        q = X[[i], :]
        q.sort_indices()
        _check(m, oracles, q, f"realtime row {i}", beam_size=5, only_topk=5)
        _check(m, oracles, q.toarray(), f"realtime dense row {i}", beam_size=5, only_topk=5)


def test_empty_and_ragged_queries(small_model):
    folder, X, m, oracles = small_model
    Xe = csr_with_empty_rows(X, [0, 3, 50, 96])
    _check(m, oracles, Xe, "empty rows", beam_size=4, only_topk=5)
    Z = smat.csr_matrix((5, X.shape[1]), dtype=np.float32)
    _check(m, oracles, Z, "all-empty batch", beam_size=4, only_topk=5)
    empty = X[:0, :]
    got = m.predict(empty, beam_size=4, only_topk=5)
    assert got.shape == (0, 300) and got.nnz == 0


def test_max_pred_chunk_tiles_equal_single_call(small_model):
    folder, X, m, oracles = small_model
    a = m.predict(X, beam_size=5, only_topk=5)
    b = m.predict(X, beam_size=5, only_topk=5, max_pred_chunk=10)
    assert_csr_parity(b, a, rtol=0.0, what="max_pred_chunk")


@pytest.mark.parametrize("permute,prune", [(True, 0.0), (False, 0.3), (True, 0.3)])
def test_non_contiguous_and_pruned_trees(tmp_path, gpu_clib, have_ref, permute, prune):
    folder = str(tmp_path / "m")
    layers = random_tree(21, [5, 40, 400], 300, 25, bias=1.0, permute=permute, prune=prune)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=6)
    X = synth.make_queries(22, 64, 300, 30)
    m, oracles = _load(folder), _oracles(folder, have_ref)
    for pp in ["l3-hinge", "noop", "log-sigmoid"]:
        _check(m, oracles, X, f"permute={permute} prune={prune}", post_processor=pp, beam_size=6, only_topk=8)
    _check(m, oracles, X[:9].toarray(), "dense", beam_size=6, only_topk=8)


def test_saturated_scores_resolve_ties_by_position(tmp_path, gpu_clib, have_ref):
    # hinge post-processors saturate to exactly 1.0 => the (parent rank, child order) tie-break decides the ids
    folder = str(tmp_path / "m")
    layers = random_tree(31, [6, 48, 600], 200, 40, bias=1.0, permute=True, saturate=True)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=10)
    X = synth.make_queries(32, 128, 200, 50)
    m, oracles = _load(folder), _oracles(folder, have_ref)
    got = _check(m, oracles, X, "saturated", beam_size=10, only_topk=10)
    assert np.mean(got.data == 1.0) > 0.2, "test is only meaningful when many scores tie"
    _check(m, oracles, X, "saturated log", post_processor="log-l3-hinge", beam_size=10, only_topk=10)


def test_no_bias_model(tmp_path, gpu_clib, have_ref):
    folder = str(tmp_path / "m")
    layers = random_tree(41, [4, 20, 150], 256, 20, bias=-1.0)
    synth.save_xlinear_model(folder, layers, bias=-1.0, only_topk=5)
    X = synth.make_queries(42, 40, 256, 30)
    m, oracles = _load(folder), _oracles(folder, have_ref)
    assert m.nr_features == 256
    _check(m, oracles, X, "no bias", beam_size=5, only_topk=5)
    _check(m, oracles, X.toarray(), "no bias dense", beam_size=5, only_topk=5)


def test_wide_chunks_long_queries_and_flat_model(tmp_path, gpu_clib, have_ref):
    # flat (depth 1) model: one chunk with 3000 columns (> shared-memory block => HBM accumulate path), more than
    # 2048 candidates (streaming top-k) and queries with more non-zeros than the shared-memory staging area.
    folder = str(tmp_path / "m")
    layers = random_tree(51, [3000], 4000, 60, bias=1.0)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=10, skip_root_C=True)
    X = synth.make_queries(52, 12, 4000, 1500)
    m, oracles = _load(folder), _oracles(folder, have_ref)
    _check(m, oracles, X, "flat k=10", only_topk=10)
    _check(m, oracles, X, "flat k=1500 (global sort path)", only_topk=1500)
    gpu_clib.clib_float32.pb200_xlinear_set_lookup(m.model.model_chain, 0)  # first-generation kernels
    _check(m, oracles, X, "flat k=10, block-wide streaming top-k + row-list streaming scores", only_topk=10)
    gpu_clib.clib_float32.pb200_xlinear_set_lookup(m.model.model_chain, 1)
    _check(m, oracles, X[:3].toarray(), "flat dense", only_topk=10)


def test_two_layer_wide_beam_streaming_topk(tmp_path, gpu_clib, have_ref):
    folder = str(tmp_path / "m")
    layers = random_tree(61, [40, 4000], 600, 20, bias=1.0)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=10)
    X = synth.make_queries(62, 30, 600, 40)
    m, oracles = _load(folder), _oracles(folder, have_ref)
    _check(m, oracles, X, "beam 40 -> 4000 candidates", beam_size=40, only_topk=25)


def test_mmap_model_equals_npz_model(tmp_path, gpu_clib, have_ref, small_model):
    """The mmap folder is written by the reference's c_xlinear_compile_mmap_model where oracle/_ref is built, else by this
    library's own (interchangeable with the reference's: tests/test_host_cpu.py, tests/golden/xlinear_toy/model_mmap)."""
    from oracle import ref

    folder, X, m, oracles = small_model
    mm_dir = str(tmp_path / "mmap_model")
    os.makedirs(mm_dir)
    if have_ref:
        ref.compile_mmap_model(os.path.join(folder, "ranker"), os.path.join(mm_dir, "ranker"))
    else:
        gpu_clib.clib_float32.c_xlinear_compile_mmap_model(os.path.join(folder, "ranker").encode(), os.path.join(mm_dir, "ranker").encode())
    mm = _load(mm_dir)
    a = m.predict(X, beam_size=5, only_topk=5)
    b = mm.predict(X, beam_size=5, only_topk=5)
    assert_csr_parity(b, a, rtol=0.0, what="mmap vs npz")
    mm_lazy = _load(mm_dir, lazy_load=True)
    assert_csr_parity(mm_lazy.predict(X, beam_size=5, only_topk=5), a, rtol=0.0, what="lazy mmap vs npz")


def test_streaming_and_lookup_kernels_agree(tmp_path, gpu_clib, have_ref):
    """The query-driven feature-map kernel and the row-list streaming kernel must return identical bits."""
    folder = str(tmp_path / "m")
    layers = random_tree(71, [6, 50, 700], 900, 35, bias=1.0, permute=True, prune=0.1)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=8)
    X = synth.make_queries(72, 150, 900, 300)
    # non-canonical CSR: repeat some column indices (only the first occurrence may count, inference.hpp:788-803)
    Xd = X.copy()
    per_row = Xd.indices.reshape(X.shape[0], -1)  # every synthetic row has the same nnz
    per_row[:, 1::7] = per_row[:, 0:-1:7][:, : per_row[:, 1::7].shape[1]]  # duplicates stay adjacent => rows stay sorted
    Xd.indices = per_row.reshape(-1)
    Xd.has_sorted_indices = True
    m, oracles = _load(folder), _oracles(folder, have_ref)
    c = gpu_clib.clib_float32
    assert c.pb200_xlinear_set_lookup(m.model.model_chain, 1) == 1
    a = _check(m, oracles, X, "lookup", beam_size=8, only_topk=10)
    a_dup = m.predict(Xd, beam_size=8, only_topk=10)
    c.pb200_xlinear_set_lookup(m.model.model_chain, 0)
    b = _check(m, oracles, X, "streaming", beam_size=8, only_topk=10)
    b_dup = m.predict(Xd, beam_size=8, only_topk=10)
    c.pb200_xlinear_set_lookup(m.model.model_chain, 2)   # feature-map lookups, one warp per chunk (no query-warp kernel)
    c2 = _check(m, oracles, X, "lookup, warp per chunk", beam_size=8, only_topk=10)
    c2_dup = m.predict(Xd, beam_size=8, only_topk=10)
    c.pb200_xlinear_set_lookup(m.model.model_chain, 3)   # query-warp kernel on every eligible layer
    c3 = _check(m, oracles, X, "query-warp kernel", beam_size=8, only_topk=10)
    c3_dup = m.predict(Xd, beam_size=8, only_topk=10)
    c.pb200_xlinear_set_lookup(m.model.model_chain, 1)
    assert_csr_parity(a, c2, rtol=0.0, what="default vs warp-per-chunk")
    assert_csr_parity(a_dup, c2_dup, rtol=0.0, what="default vs warp-per-chunk, duplicated column indices")
    assert_csr_parity(a, c3, rtol=0.0, what="default vs query-warp")
    assert_csr_parity(a_dup, c3_dup, rtol=0.0, what="default vs query-warp, duplicated column indices")
    assert_csr_parity(a, b, rtol=0.0, what="lookup vs streaming")
    assert_csr_parity(a_dup, b_dup, rtol=0.0, what="lookup vs streaming, duplicated column indices")
    if "reference" in oracles:
        assert_csr_parity(a_dup, oracles["reference"].predict(Xd, 8, None, 10), what="duplicated column indices vs reference")


def test_resident_batch_and_counters(small_model, gpu_clib):
    """Device-resident path used by bench.py: same answers, plus algorithmic-byte counters and launch counts."""
    from ctypes import byref, c_double, c_uint64

    from pecos_b200.core import ScipyCompressedSparseAllocator, ScipyCsrF32

    folder, X, m, oracles = small_model
    c = gpu_clib.clib_float32
    h = m.model.model_chain
    cx = ScipyCsrF32.init_from(X)
    c.pb200_xlinear_resident_upload_csr(h, byref(cx))
    ms = c.pb200_xlinear_resident_predict(h, 5, None, 5, 1)
    assert ms > 0
    alloc = ScipyCompressedSparseAllocator()
    c.pb200_xlinear_resident_fetch(h, alloc.cfunc)
    assert_csr_parity(alloc.get(), m.predict(X, beam_size=5, only_topk=5), rtol=0.0, what="resident")
    stats = (c_uint64 * (7 * 3))()
    c.pb200_xlinear_get_stats(h, stats)
    s = np.array(list(stats), dtype=np.int64).reshape(3, 7)
    assert s[0, 0] == X.shape[0]             # layer 0: one chunk (the root) per query
    assert s[1, 0] == 4 * X.shape[0]         # layer 1: beam = all 4 root children
    assert s[2, 0] == 5 * X.shape[0]         # layer 2: beam_size chunks per query
    assert (s[:, 2] >= s[:, 0]).all()        # every chunk applies at least its bias row
    assert c.pb200_xlinear_launches(h) > 0


def test_eurlex_shaped_sample_matches_reference(tmp_path, gpu_clib, have_ref):
    """BASELINE.json configs[1] shape (L=3956, D=5000, layers 4/64/3956, beam 10, top-10) on a 600-query sample."""
    folder = str(tmp_path / "eurlex")
    _, X, cfg = synth.build_workload("eurlex-4k", folder, scale_queries=600)
    m, oracles = _load(folder), _oracles(folder, have_ref)
    if "reference" in oracles:
        oracles = {"reference": oracles["reference"]}  # the scalar restatement is slow at this width
    got = _check(m, oracles, X, "eurlex-4k", beam_size=cfg["beam_size"], only_topk=cfg["only_topk"])
    assert (got.getnnz(axis=1) == 10).all()


@pytest.mark.parametrize("scale", [1.0, 8.0, 60.0])
def test_topk_estimate_filter_is_exact(tmp_path, gpu_clib, have_ref, scale):
    """xl_topk_filter_kernel (single-precision estimates pick the candidates that get the exact post-processor) must return
    the bits of the kernel that evaluates every candidate (kernel mode 4) and of the oracles: plain, saturated (hundreds
    of exact ties) and extreme (exp under/overflow, log-sigmoid asymptote) score ranges, wide rows (> 32 survivors per
    batch), k = 32 (the filter's limit) and k = 33 (falls back)."""
    folder = str(tmp_path / "m")
    layers = random_tree(81, [8, 64, 2400], 700, 30, bias=1.0, permute=True)
    layers = [(smat.csc_matrix(W * np.float32(scale), dtype=np.float32), C) for W, C in layers]
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=10)
    X = synth.make_queries(82, 160, 700, 60)
    m, oracles = _load(folder), _oracles(folder, have_ref)
    c = gpu_clib.clib_float32
    for pp in POST_PROCESSORS:
        for beam, topk in [(10, 10), (32, 32), (20, 33), (64, 7)]:
            if pp not in ("l3-hinge", "log-l3-hinge", "sigmoid") and (beam, topk) != (10, 10):
                continue
            c.pb200_xlinear_set_lookup(m.model.model_chain, 1)
            a = _check(m, oracles, X, f"filter scale={scale}", post_processor=pp, beam_size=beam, only_topk=topk)
            c.pb200_xlinear_set_lookup(m.model.model_chain, 4)
            b = m.predict(X, post_processor=pp, beam_size=beam, only_topk=topk)
            assert_csr_parity(a, b, rtol=0.0, what=f"filter vs evaluate-all {pp} beam={beam} k={topk} scale={scale}")
    c.pb200_xlinear_set_lookup(m.model.model_chain, 1)


def test_pipelined_uploads_equal_unpipelined_calls(small_model):
    """Batches of >= 4096 rows are cut into sub-tiles whose host->device copies overlap the scoring of the previous
    sub-tile (two staging sets, copy stream).  Same bits as calls small enough not to be pipelined, and as the oracle;
    ragged rows make the sub-tiles uneven."""
    folder, X, m, oracles = small_model
    big = smat.vstack([X] * 60, format="csr").astype(np.float32)[:5531]
    big = csr_with_empty_rows(big, [0, 1, 4095, 4096, 5530])
    a = _check(m, {"restatement": oracles["restatement"]}, big, "pipelined", beam_size=6, only_topk=5)
    b = m.predict(big, beam_size=6, only_topk=5, max_pred_chunk=1000)
    assert_csr_parity(a, b, rtol=0.0, what="pipelined vs small calls")
    a2 = m.predict(big, beam_size=6, only_topk=5)  # staging sets are reused by the next call
    assert_csr_parity(a2, a, rtol=0.0, what="second pipelined call")


# ------------------------------------------------------------------------------------------------ reference goldens
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "xlinear_toy")


def test_reference_golden_vectors_through_the_cuda_path(gpu_clib):
    """All 90 entries recorded FROM THE REFERENCE (tests/golden/make_golden.py: 3 models x 15 (post-processor, beam, top-k)
    settings x csr/dense queries on the reference's own toy fixture) through the CUDA engine: ids and ranks bit-exact,
    scores within 1e-5 relative.  Needs no oracle at test time."""
    import json

    E = np.load(os.path.join(GOLD, "expected.npz"))
    index = json.load(open(os.path.join(GOLD, "expected_index.json")))
    Xt = smat.load_npz(os.path.join(GOLD, "Xt.npz")).tocsr().astype(np.float32)
    Xt.sort_indices()
    models, n = {}, 0
    for item in index:
        name = item["model"]
        m = models.get(name) or models.setdefault(name, _load(os.path.join(GOLD, name)))
        Xq = Xt if item["kind"] == "csr" else np.ascontiguousarray(Xt.toarray())
        kw = {}
        if item["post_processor"]:
            kw["post_processor"] = item["post_processor"]
        if item["beam_size"]:
            kw["beam_size"] = item["beam_size"]
        if item["only_topk"]:
            kw["only_topk"] = item["only_topk"]
        got = m.predict(Xq, **kw)
        key = item["key"]
        want = smat.csr_matrix((E[key + "|data"], E[key + "|indices"], E[key + "|indptr"]), shape=tuple(item["shape"]))
        assert_csr_parity(got, want, what=key)
        n += 1
    assert n == len(index) and n >= 90


def test_reference_compiled_mmap_model_through_the_cuda_path(gpu_clib):
    """tests/golden/xlinear_toy/model_mmap was written by the REFERENCE's c_xlinear_compile_mmap_model; loading it through
    c_xlinear_load_mmap_model_from_disk (eager and lazy) must reproduce the recorded reference predictions
    (test/pecos/xmc/xlinear/test_xlinear.py:1140-1168)."""
    import json

    E = np.load(os.path.join(GOLD, "expected.npz"))
    index = [it for it in json.load(open(os.path.join(GOLD, "expected_index.json"))) if it["model"] == "model" and it["kind"] == "csr"]
    Xt = smat.load_npz(os.path.join(GOLD, "Xt.npz")).tocsr().astype(np.float32)
    Xt.sort_indices()
    for lazy in (False, True):
        m = _load(os.path.join(GOLD, "model_mmap"), lazy_load=lazy)
        for item in index:
            kw = {k: item[k] for k in ("post_processor", "beam_size", "only_topk") if item[k]}
            key = item["key"]
            want = smat.csr_matrix((E[key + "|data"], E[key + "|indices"], E[key + "|indptr"]), shape=tuple(item["shape"]))
            assert_csr_parity(m.predict(Xt, **kw), want, what=f"mmap lazy={lazy} {key}")
    gold = np.load(os.path.join(GOLD, "Yt_pred_reference_golden.npy"))  # the reference repo's own Yt_pred.npz
    assert np.abs(_load(os.path.join(GOLD, "model_mmap")).predict(Xt).toarray() - gold).max() <= 1e-6


def test_synthetic_3m_slice_matches_the_recorded_reference_result(gpu_clib, tmp_path_factory):
    """BASELINE.json configs[2] at FULL size (3M labels, 500k features, depth 6, beam 20, top-10): the first 2,000 queries of the
    benchmark batch against the result RECORDED FROM THE REFERENCE LIBRARY (tests/golden/make_golden_s_slice.py; no oracle/_ref
    needed here).  The model is regenerated from the same seeds (pecos_b200/synth.py) -- reusing bench.py's cache folder when it
    exists on this box (~1.5 min otherwise).  ids / ranks bit-exact, scores 1e-5."""
    import tempfile

    gold = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "synthetic3m_slice", "expected.npz")
    E = np.load(gold)
    folder = os.path.join(os.environ.get("PB200_BENCH_CACHE", os.path.join(tempfile.gettempdir(), "pecos_b200_bench")), "synthetic-3m")
    synth.build_workload("synthetic-3m", folder, scale_queries=8)  # writes the model if absent
    cfg = synth.WORKLOADS["synthetic-3m"]
    assert int(E["query_seed"]) == cfg["query_seed"]
    X = synth.make_queries(cfg["query_seed"], int(E["query_rows"]), cfg["D"], cfg["nnz_per_row"], synth.zipf_cdf(cfg["D"]))
    m = _load(folder)
    got = m.predict(X, beam_size=cfg["beam_size"], only_topk=cfg["only_topk"])
    want = smat.csr_matrix((E["data"], E["indices"].astype(np.int64), E["indptr"]), shape=(X.shape[0], cfg["layer_sizes"][-1]))
    assert_csr_parity(got, want, what="synthetic-3m slice vs recorded reference")
