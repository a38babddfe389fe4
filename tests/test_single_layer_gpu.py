"""GPU parity tests for the next scope row (SURVEY 8f-2): c_xlinear_single_layer_predict_{csr,drm}_f32, the per-layer
entry point of the reference's python prediction chain (pecos/core/libpecos.cpp:201-235, pecos/xmc/base.py:890-949).

The oracle is pinned by
tests/test_oracle_cpu.py::test_single_layer_restatement_equals_reference_library.
"""
import os
from ctypes import c_uint64

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .util import RecordedReference, assert_csr_parity, random_tree

pytestmark = pytest.mark.gpu


def _oracle_single(have_ref):
    from oracle import ref, restatement

    fns = {"restatement": restatement.single_layer_predict}
    if have_ref:
        fns["reference"] = ref.single_layer_predict
    return fns


def _shuffle_rows(M, seed, empty=()):
    rng = np.random.default_rng(seed)
    lil = M.tolil()
    for r in empty:
        lil.rows[r], lil.data[r] = [], []
    out = lil.tocsr().astype(np.float32)
    for r in range(out.shape[0]):
        s, e = out.indptr[r], out.indptr[r + 1]
        perm = rng.permutation(e - s)
        out.indices[s:e] = out.indices[s:e][perm]
        out.data[s:e] = out.data[s:e][perm]
    out.has_sorted_indices = False
    return out


@pytest.mark.parametrize("permute,prune", [(False, 0.0), (True, 0.25)])
def test_single_layer_matches_the_oracles(gpu_clib, have_ref, permute, prune):
    from pecos_b200.xlinear import MLModel

    layers = random_tree(101, [5, 30, 240], 150, 20, bias=1.0, permute=permute, prune=prune)
    X = synth.make_queries(102, 40, 150, 25)
    oracles = _oracle_single(have_ref)
    prev = None
    for d, (W, C) in enumerate(layers):
        m = MLModel(W, C, bias=1.0)
        for pp in ["l3-hinge", "noop", "sigmoid", "log-sigmoid", "log-l2-hinge"]:
            for Xq, codes in ((X, prev), (X[:7].toarray(), None if prev is None else prev[:7])):
                got = m.predict(Xq, csr_codes=codes, only_topk=6, post_processor=pp)
                for name, fn in oracles.items():
                    want = fn(Xq, codes, W, C, pp, 6, 1.0)
                    assert_csr_parity(got, want, what=f"layer {d} {pp} vs {name}")
        prev = m.predict(X, csr_codes=prev, only_topk=4, post_processor="l3-hinge")
        if d + 1 < len(layers):
            Wn, Cn = layers[d + 1]
            shuffled = _shuffle_rows(prev, 103 + d, empty=(3, 11))  # the beam is consumed in stored order
            got = MLModel(Wn, Cn, bias=1.0).predict(X, csr_codes=shuffled, only_topk=6, post_processor="l3-hinge")
            for name, fn in oracles.items():
                assert_csr_parity(got, fn(X, shuffled, Wn, Cn, "l3-hinge", 6, 1.0), what=f"layer {d + 1} shuffled codes vs {name}")


def test_python_chain_equals_predict_only_model(tmp_path, gpu_clib, have_ref):
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    layers = random_tree(111, [6, 48, 500], 300, 30, bias=1.0, permute=True)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=8)
    X = synth.make_queries(112, 64, 300, 40)
    fast = XLinearModel.load(folder, is_predict_only=True)
    chain = XLinearModel.load(folder, is_predict_only=False)
    assert not chain.is_predict_only and chain.depth == 3 and chain.nr_labels == 500
    for kw in (dict(beam_size=5, only_topk=8), dict(beam_size=10, only_topk=3, post_processor="sigmoid")):
        assert_csr_parity(chain.predict(X, **kw), fast.predict(X, **kw), rtol=0.0, what=f"chain vs predict-only {kw}")
    assert_csr_parity(chain.predict(X.toarray()[:9], beam_size=5, only_topk=8), fast.predict(X.toarray()[:9], beam_size=5, only_topk=8),
                      rtol=0.0, what="dense chain vs predict-only")


def test_layer_cache_and_edge_cases(gpu_clib, have_ref):
    from pecos_b200.xlinear import MLModel

    c = gpu_clib.clib_float32
    c.pb200_layer_cache_clear()
    info = (c_uint64 * 3)()
    c.pb200_layer_cache_info(info)
    misses0 = int(info[2])
    (W, C), = random_tree(121, [40], 120, 15, bias=1.0)
    X = synth.make_queries(122, 20, 120, 20)
    m = MLModel(W, C, bias=1.0)
    a = m.predict(X, only_topk=5, post_processor="l3-hinge")
    b = m.predict(X, only_topk=5, post_processor="l3-hinge")  # second call: same engine
    assert_csr_parity(a, b, rtol=0.0, what="cached layer")
    c.pb200_layer_cache_info(info)
    assert int(info[0]) == 1 and int(info[2]) == misses0 + 1 and int(info[1]) >= 1
    W2 = W.copy()
    W2.data[::7] *= np.float32(1.5)  # other weights, same shape: another engine, other scores
    a2 = MLModel(W2, C, bias=1.0).predict(X, only_topk=5, post_processor="l3-hinge")
    c.pb200_layer_cache_info(info)
    assert int(info[0]) == 2
    assert not np.array_equal(a.data, a2.data)
    for name, fn in _oracle_single(have_ref).items():
        assert_csr_parity(a2, fn(X, None, W2, C, "l3-hinge", 5, 1.0), what=f"second layer vs {name}")
    from pecos_b200.xlinear import MLModelPredParams

    empty = m.predict(X, pred_params=MLModelPredParams(only_topk=0, post_processor="l3-hinge"))  # sorted_csr keeps min(nnz, 0)
    assert empty.shape == (20, 40) and empty.nnz == 0
    none = m.predict(X[:0, :], only_topk=5, post_processor="l3-hinge")
    assert none.shape == (0, 40) and none.nnz == 0
    assert c.pb200_layer_cache_clear() == 2


@pytest.mark.parametrize("permute,prune", [(False, 0.0), (True, 0.2)])
def test_single_layer_selected_outputs_equal_the_reference_library(gpu_clib, have_ref, permute, prune):
    """c_xlinear_single_layer_predict_on_selected_outputs_{csr,drm}_f32 (libpecos.cpp:238-273; the per-layer call of
    predict_on_selected_outputs for is_predict_only=False models, pecos/xmc/base.py:1003): the pattern of the selection, values =
    transformed (+ combined) scores -- ids bit-exact, scores 1e-5 vs the reference library on the same W / C / codes (its
    recorded results where oracle/_ref is not built)."""
    from oracle import ref

    rec = RecordedReference(f"single_layer_selected_{int(permute)}_{int(prune > 0)}", have_ref)

    layers = random_tree(411, [5, 40, 500], 300, 20, bias=1.0, permute=permute, prune=prune)
    X = synth.make_queries(412, 300, 300, 30)
    rng = np.random.default_rng(413)
    g = gpu_clib.clib_float32
    for d in (1, 2):
        W, C = layers[d]
        Cr = smat.csr_matrix(C)
        n_labels, n_codes = C.shape
        has_parent = np.asarray(Cr.sum(axis=1)).ravel() > 0  # a parentless label is outside the reference's contract (it reads out of bounds)
        sel = smat.csr_matrix(((rng.random((300, n_labels)) < 0.04) & has_parent[None, :]).astype(np.float32))
        pattern = ((sel @ Cr) + smat.csr_matrix((rng.random((300, n_codes)) < 0.1).astype(np.float32))).tocsr()
        pattern.sort_indices()
        codes = smat.csr_matrix((0.05 + rng.random(pattern.nnz).astype(np.float32), pattern.indices, pattern.indptr), shape=pattern.shape)
        for pp in ("l3-hinge", "sigmoid", "log-l2-hinge", "noop"):
            for cc in ((codes, None) if d == 1 else (codes,)):
                for Xq in (X, np.ascontiguousarray(X.toarray()[:40])):
                    c2 = cc if cc is None or Xq is X else cc[:40]
                    s2 = sel if Xq is X else sel[:40]
                    got = ref.single_layer_predict_on_selected_outputs(Xq, s2, c2, W, C, pp, 1.0, clib=g)
                    rec.check(f"{d}|{pp}|{cc is not None}|{Xq is X}", got,
                              lambda: ref.single_layer_predict_on_selected_outputs(Xq, s2, c2, W, C, pp, 1.0),
                              what=f"single-layer selected d={d} {pp} codes={cc is not None}")
    rec.close()
