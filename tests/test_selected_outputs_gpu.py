"""GPU parity tests for c_xlinear_predict_on_selected_outputs_{csr,drm}_f32 (pecos/core/libpecos.cpp:179-198; SURVEY 8f-2).

CUDA path (XLinearEngine::predict_selected in pecos_b200/csrc/xlinear_engine.cu) vs the C restatement (pinned bit-for-bit against the reference library in
tests/test_oracle_cpu.py) and, where oracle/_ref is present, vs the reference library itself (CSC handle).  Bar: same entry
order and label ids, scores 1e-5 relative.  Mirrors test/pecos/xmc/xlinear/test_xlinear.py:1059-1137.
"""
import os

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .util import assert_csr_parity, random_tree, reachable_labels

pytestmark = pytest.mark.gpu


def _selection(rng, rows, n_labels, max_per_row, allowed=None):
    allowed = np.arange(n_labels) if allowed is None else np.asarray(allowed)
    r, c = [], []
    for q in range(rows):
        k = int(rng.integers(0, max_per_row + 1))  # some rows select nothing
        cols = rng.choice(allowed, size=min(k, allowed.size), replace=False)
        r += [q] * len(cols)
        c += list(cols)  # unsorted on purpose: the reference sorts the leaf set itself
    return smat.csr_matrix((np.ones(len(r), dtype=np.float32), (r, c)), shape=(rows, n_labels))


@pytest.mark.parametrize("permute,prune,sizes", [(False, 0.0, [6, 40, 300]), (True, 0.0, [6, 40, 300]), (True, 0.25, [5, 30, 400]),
                                                 (False, 0.0, [50])])
def test_selected_outputs_equal_the_oracles(tmp_path, gpu_clib, have_ref, permute, prune, sizes):
    from oracle import restatement
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    layers = random_tree(95, sizes, 200, 25, bias=1.0, permute=permute, prune=prune)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=6)
    X = synth.make_queries(96, 300, 200, 30)
    # pruned trees: only labels with a path to the root (the reference indexes with uninitialised memory otherwise)
    S = _selection(np.random.default_rng(97), 300, sizes[-1], 12, allowed=reachable_labels(layers))
    # the reference serves selected outputs from CSC handles (whose nr_labels = W.cols also on pruned trees): load the same way
    m = XLinearModel.load(folder, is_predict_only=True, weight_matrix_type="CSC")
    assert m.nr_labels == sizes[-1]
    o = restatement.OracleXLinear(os.path.join(folder, "ranker"))
    r = None
    if have_ref:
        from oracle import ref

        r = ref.RefXLinear(os.path.join(folder, "ranker"), weight_matrix_type="CSC")
    for pp in [None, "noop", "sigmoid", "log-sigmoid", "l2-hinge", "log-l3-hinge"]:
        for Xq, Sq in ((X, S), (np.ascontiguousarray(X.toarray()[:40]), S[:40])):
            kw = {"post_processor": pp} if pp else {}
            got = m.predict(Xq, selected_outputs_csr=Sq, **kw)
            assert got.nnz == Sq.nnz
            assert_csr_parity(got, o.predict_on_selected_outputs(Xq, Sq, pp), what=f"vs restatement {pp}")
            if r is not None:
                from oracle import ref

                assert_csr_parity(got, ref.predict_on_selected_outputs(r, Xq, Sq, pp), what=f"vs reference {pp}")
    # chunked calls (max_pred_chunk) concatenate to the same matrix
    assert_csr_parity(m.predict(X, selected_outputs_csr=S, max_pred_chunk=77), m.predict(X, selected_outputs_csr=S), rtol=0.0,
                      what="max_pred_chunk")


def test_unreachable_selected_labels_leave_zero_entries(tmp_path, gpu_clib):
    """Pruned tree, selection includes labels WITHOUT a path to the root: out of the reference's contract (it reads
    uninitialised memory); the CUDA path and the restatement both leave zero entries at the end of such rows."""
    from oracle import restatement
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    layers = random_tree(395, [5, 30, 400], 200, 25, bias=1.0, permute=True, prune=0.3)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=6)
    X = synth.make_queries(396, 120, 200, 30)
    S = _selection(np.random.default_rng(397), 120, 400, 15)
    assert np.setdiff1d(np.unique(S.indices), reachable_labels(layers)).size > 0
    m = XLinearModel.load(folder, is_predict_only=True, weight_matrix_type="CSC")
    o = restatement.OracleXLinear(os.path.join(folder, "ranker"))
    assert_csr_parity(m.predict(X, selected_outputs_csr=S), o.predict_on_selected_outputs(X, S, None), what="unreachable labels")


def test_selected_scores_equal_beam_search_scores(tmp_path, gpu_clib):
    """A label returned by beam search has the same score BITS when it is selected explicitly (same kernels, same order)."""
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    layers = random_tree(195, [6, 40, 300], 200, 25, bias=1.0)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=6)
    X = synth.make_queries(196, 500, 200, 30)
    m = XLinearModel.load(folder, is_predict_only=True)
    full = m.predict(X, beam_size=40, only_topk=5)  # beam 40 = exhaustive at the middle layer
    sel = m.predict(X, selected_outputs_csr=smat.csr_matrix(full, dtype=np.float32))
    assert np.array_equal(full.toarray().view(np.uint32), sel.toarray().view(np.uint32))


def test_selected_outputs_argument_checks(tmp_path, gpu_clib):
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, random_tree(5, [4, 30], 50, 8, bias=1.0), bias=1.0, only_topk=3)
    m = XLinearModel.load(folder, is_predict_only=True)
    X = synth.make_queries(6, 10, 50, 5)
    with pytest.raises(ValueError):
        m.predict(X, selected_outputs_csr=smat.csr_matrix((10, 31), dtype=np.float32))
    with pytest.raises(ValueError):
        m.predict(X, selected_outputs_csr=smat.csr_matrix((9, 30), dtype=np.float32))
    with pytest.raises(ValueError):
        m.predict(X, selected_outputs_csr=np.zeros((10, 30), dtype=np.float32))
    empty = m.predict(X, selected_outputs_csr=smat.csr_matrix((10, 30), dtype=np.float32))
    assert empty.nnz == 0 and empty.shape == (10, 30)


@pytest.mark.parametrize("permute,prune", [(False, 0.0), (True, 0.2)])
def test_python_chain_selected_outputs_equal_predict_only_and_reference(tmp_path, gpu_clib, have_ref, permute, prune):
    """is_predict_only=False models (list of MLModel, one c_xlinear_single_layer_predict_on_selected_outputs_* call per layer,
    pecos/xmc/base.py:1772-1793) score a selection exactly like the predict-only handle and like the reference library."""
    from pecos_b200.xlinear import XLinearModel

    from .util import reachable_labels

    folder = str(tmp_path / "m")
    layers = random_tree(511, [6, 40, 400], 250, 22, bias=1.0, permute=permute, prune=prune)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=6, post_processor="l3-hinge")
    X = synth.make_queries(512, 300, 250, 28)
    rng = np.random.default_rng(513)
    ok = np.zeros(layers[-1][0].shape[1], dtype=bool)
    ok[reachable_labels(layers)] = True
    sel = smat.csr_matrix(((rng.random((300, ok.size)) < 0.03) & ok[None, :]).astype(np.float32))
    chain = XLinearModel.load(folder, is_predict_only=False)
    handle = XLinearModel.load(folder, is_predict_only=True, weight_matrix_type="CSC")
    for pp in (None, "sigmoid", "log-l2-hinge"):
        kw = {} if pp is None else {"post_processor": pp}
        for Xq, s in ((X, sel), (np.ascontiguousarray(X.toarray()[:50]), sel[:50])):
            got = chain.predict(Xq, selected_outputs_csr=s, **kw)
            want = handle.predict(Xq, selected_outputs_csr=s, **kw)
            assert_csr_parity(got, want, what=f"python chain vs predict-only handle ({pp})")
            if have_ref:
                from oracle import ref

                r = ref.RefXLinear(os.path.join(folder, "ranker"), weight_matrix_type="CSC")
                assert_csr_parity(got, ref.predict_on_selected_outputs(r, Xq, s, pp), what=f"python chain vs reference library ({pp})")
