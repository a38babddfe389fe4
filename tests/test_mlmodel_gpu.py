"""GPU parity tests for the single-layer mmap handle API c_mlmodel_* (pecos/core/libpecos.cpp:37-113; SURVEY 8f-2).

* tests/golden/mlmodel_toy: a single-layer mmap folder written by the REFERENCE (c_mlmodel_compile_mmap_model) + 48 recorded
  reference results (c_mlmodel_predict_* and c_mlmodel_predict_on_selected_outputs_*, csr / dense queries, with and without
  csr_codes, four post-processors) -- needs no oracle at test time;
* random layers: the CUDA library and the reference library are driven through the SAME ctypes wrapper (oracle/ref.py
  MLModelHandle) on folders compiled by the reference here.
Bar: ids / ranks bit-exact, scores 1e-5 relative."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .util import RecordedReference, assert_csr_parity, random_tree

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "mlmodel_toy")
TOY = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "xlinear_toy")


def test_reference_golden_results_through_the_cuda_path(gpu_clib):
    from oracle.ref import MLModelHandle  # the ctypes wrapper only: nothing of oracle/ is executed here

    c = gpu_clib.clib_float32
    m = MLModelHandle(os.path.join(GOLD, "layer_mmap"), clib=c)
    ml = MLModelHandle(os.path.join(GOLD, "layer_mmap"), clib=c, lazy_load=True)
    meta = json.load(open(os.path.join(GOLD, "expected_index.json")))
    for k, v in meta["attrs"].items():
        assert m.attr(k) == v
    E = np.load(os.path.join(GOLD, "expected.npz"))
    Xt = smat.load_npz(os.path.join(TOY, "Xt.npz")).tocsr().astype(np.float32)
    Xt.sort_indices()
    codes = smat.load_npz(os.path.join(GOLD, "codes.npz")).tocsr()
    sel = smat.load_npz(os.path.join(GOLD, "selected.npz")).tocsr()
    n = 0
    for it in meta["entries"]:
        Xq = Xt if it["kind"] == "csr" else np.ascontiguousarray(Xt.toarray())
        cc = codes if it["codes"] == "codes" else None
        key = it["key"]
        want = smat.csr_matrix((E[key + "|data"], E[key + "|indices"], E[key + "|indptr"]), shape=tuple(it["shape"]))
        for h in (m, ml):
            if it["op"] == "predict":
                got = h.predict(Xq, cc, it["post_processor"], it["only_topk"])
            else:
                got = h.predict_on_selected_outputs(Xq, sel, cc, it["post_processor"])
            assert_csr_parity(got, want, what=key)
        n += 1
    assert n == 48


@pytest.mark.parametrize("permute,prune", [(False, 0.0), (True, 0.2)])
def test_random_layers_equal_the_reference_library(tmp_path, gpu_clib, have_ref, permute, prune):
    """Where oracle/_ref is not built, the reference's recorded results stand in for it, and the mmap folder is written by this
    library's own c_mlmodel_compile_mmap_model (interchangeable with the reference's: tests/test_host_cpu.py)."""
    from oracle import ref

    rec = RecordedReference(f"mlmodel_random_{int(permute)}_{int(prune > 0)}", have_ref)

    folder = str(tmp_path / "m")
    layers = random_tree(311, [5, 40, 600], 300, 20, bias=1.0, permute=permute, prune=prune)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=7, post_processor="l2-hinge")
    X = synth.make_queries(312, 400, 300, 30)
    rng = np.random.default_rng(313)
    for d in (1, 2):
        mm = str(tmp_path / f"ml{d}")
        ref.compile_mlmodel_mmap(os.path.join(folder, "ranker", f"{d}.model"), mm, clib=None if have_ref else gpu_clib.clib_float32)
        r = ref.MLModelHandle(mm) if have_ref else None
        g = ref.MLModelHandle(mm, clib=gpu_clib.clib_float32)
        n_labels, n_codes = layers[d][1].shape
        assert (g.attr("nr_codes"), g.attr("nr_labels"), g.attr("nr_features")) == (n_codes, n_labels, 300)
        if r is not None:
            assert (r.attr("nr_codes"), r.attr("nr_labels"), r.attr("nr_features")) == (n_codes, n_labels, 300)
        C = smat.load_npz(os.path.join(folder, "ranker", f"{d}.model", "C.npz")).tocsr()
        has_parent = np.asarray(C.sum(axis=1)).ravel() > 0   # pruned trees: a parentless label is outside the reference's contract
        sel = smat.csr_matrix(((rng.random((400, n_labels)) < 0.03) & has_parent[None, :]).astype(np.float32))
        # csr_codes = parents of the selected labels (what the reference's callers pass: selected x C, pecos/xmc/base.py:1771-1780;
        # the reference reads out of bounds when a selected label's parent is missing) + some extra codes
        pattern = ((sel @ C) + smat.csr_matrix((rng.random((400, n_codes)) < 0.1).astype(np.float32))).tocsr()
        pattern.sort_indices()
        codes = smat.csr_matrix((0.05 + rng.random(pattern.nnz).astype(np.float32), pattern.indices, pattern.indptr), shape=pattern.shape)
        for pp in (None, "sigmoid", "log-l3-hinge"):
            for cc in (codes, None) if d == 1 else (codes,):  # "no codes" on the 600-label layer = 40 x 600 candidates: covered at d = 1
                for Xq in (X, np.ascontiguousarray(X.toarray()[:50])):
                    c2 = cc if cc is None or Xq is X else cc[:50]
                    s2 = sel if Xq is X else sel[:50]
                    key = f"{d}|{pp}|{cc is not None}|{Xq is X}"
                    for topk in (0, 4):
                        rec.check(f"{key}|predict|{topk}", g.predict(Xq, c2, pp, topk), lambda: r.predict(Xq, c2, pp, topk),
                                  what=f"predict d={d} {pp} k={topk}")
                    rec.check(f"{key}|selected", g.predict_on_selected_outputs(Xq, s2, c2, pp),
                              lambda: r.predict_on_selected_outputs(Xq, s2, c2, pp), what=f"selected d={d} {pp}")
    rec.close()
