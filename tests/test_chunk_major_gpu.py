"""GPU tests for the chunk-major score kernel (pecos_b200/csrc/xlinear_cm_kernel.cuh): the default scorer wherever a layer's
feature map + largest chunk fit in shared memory.  It must return the same BITS as the query-major kernels (kernel mode 6
switches it off) and match both oracles (ids bit-exact, scores 1e-5)."""
import os
from ctypes import c_int

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .util import assert_csr_parity, csr_with_empty_rows, random_tree

pytestmark = pytest.mark.gpu


def _oracles(folder, have_ref):
    from oracle import ref, restatement

    out = {"restatement": restatement.OracleXLinear(os.path.join(folder, "ranker"))}
    if have_ref:
        out["reference"] = ref.RefXLinear(os.path.join(folder, "ranker"))
    return out


@pytest.mark.parametrize("permute,prune,sizes,bias", [(False, 0.0, [8, 64, 512], 1.0), (True, 0.2, [8, 64, 512], 1.0),
                                                      (False, 0.0, [4, 24, 1500], 1.0),   # wide chunks (~62 columns, eurlex-like)
                                                      (True, 0.1, [6, 300], -1.0),        # no bias row
                                                      (False, 0.0, [2, 4, 1800], 1.0)])   # 450-column chunks (> 256): cut into column ranges
def test_chunk_major_kernel_equals_default_kernels_and_oracles(tmp_path, gpu_clib, have_ref, permute, prune, sizes, bias):
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    # enough queries that every chunk is visited by >= 24 pairs on average
    layers = random_tree(131, sizes, 400, 24, bias=bias, permute=permute, prune=prune)
    synth.save_xlinear_model(folder, layers, bias=bias, only_topk=8)
    X = synth.make_queries(132, 3000, 400, 48)
    X = csr_with_empty_rows(X, [0, 7, 2999])
    # repeated column indices: only the first occurrence counts (inference.hpp:788-803)
    Xd = X.copy()
    for r in (3, 11, 500):
        s, e = Xd.indptr[r], Xd.indptr[r + 1]
        if e - s >= 4:
            Xd.indices[s + 1] = Xd.indices[s]
            Xd.indices[s + 3] = Xd.indices[s + 2]
    Xd.has_sorted_indices = True
    Xl = synth.make_queries(133, 200, 400, 300)  # long rows: many rounds of the staging ring
    m, oracles = XLinearModel.load(folder, is_predict_only=True), _oracles(folder, have_ref)
    c = gpu_clib.clib_float32
    h = m.model.model_chain
    for pp in ("l3-hinge", "noop", "log-sigmoid"):
        for Xq in (X, Xd, Xl):
            c.pb200_xlinear_set_lookup(h, 6)
            base = m.predict(Xq, beam_size=10, only_topk=8, post_processor=pp)
            kid = (c_int * 6)()
            c.pb200_xlinear_get_kernel_ids(h, kid)
            assert 4 not in [kid[2 * d] for d in range(len(sizes))], "kernel mode 6 must not use the chunk-major kernel"
            c.pb200_xlinear_set_lookup(h, 5)  # chunk-major wherever it fits (mode 1 also asks for >= 148 work items)
            got = m.predict(Xq, beam_size=10, only_topk=8, post_processor=pp)
            c.pb200_xlinear_get_kernel_ids(h, kid)
            assert all(kid[2 * d] == 4 for d in range(len(sizes))), "the chunk-major kernel must serve every layer of this model"
            assert_csr_parity(got, base, rtol=0.0, what=f"chunk-major vs default {pp}")
            if Xq is X:
                for name, o in oracles.items():
                    sub = slice(0, 200)
                    assert_csr_parity(got[sub], o.predict(Xq[sub], 10, pp, 8), what=f"chunk-major vs {name} {pp}")
    c.pb200_xlinear_set_lookup(h, 1)


def test_chunk_major_tiles_and_small_batches(tmp_path, gpu_clib, have_ref):
    """Few queries => the reuse heuristic keeps the default kernels; max_pred_chunk tiles re-run the bucketing per call."""
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    layers = random_tree(141, [8, 64, 512], 300, 20, bias=1.0)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=6)
    X = synth.make_queries(142, 2500, 300, 40)
    m = XLinearModel.load(folder, is_predict_only=True)
    c = gpu_clib.clib_float32
    h = m.model.model_chain
    c.pb200_xlinear_set_lookup(h, 6)
    base = m.predict(X, beam_size=8, only_topk=6)
    c.pb200_xlinear_set_lookup(h, 5)
    assert_csr_parity(m.predict(X, beam_size=8, only_topk=6, max_pred_chunk=1300), base, rtol=0.0, what="tiled")
    c.pb200_xlinear_set_lookup(h, 1)
    small = m.predict(X[:5], beam_size=8, only_topk=6)
    kid = (c_int * 6)()
    c.pb200_xlinear_get_kernel_ids(h, kid)
    assert kid[4] != 4, "5 queries x beam 8 must not pay for staging 512 chunks"
    assert_csr_parity(small, base[:5], rtol=0.0, what="small batch")
    c.pb200_xlinear_set_lookup(h, 1)

