"""GPU tests of the prefix kernel: layers 0 and 1 scored by ONE chunk-major launch over their merged image, layer 0's beam
chosen in the same kernel.  Kernel mode 7 switches it off; both must return the same ids, counts and score BITS."""
import json
import os
from ctypes import byref, c_double

import numpy as np
import pytest

from pecos_b200 import synth

from .util import assert_csr_parity, csr_with_empty_rows, random_tree

pytestmark = pytest.mark.gpu


def _same_bits(got, want, what):
    assert_csr_parity(got, want, rtol=0.0, what=what)
    assert np.array_equal(np.asarray(got.data, dtype=np.float32).view(np.uint32),
                          np.asarray(want.data, dtype=np.float32).view(np.uint32)), f"{what}: score bits differ"


def _profile(c, h, depth, run):
    """Runs run() with per-layer event timing; True when the prefix served the call (layer 0's top-k slot and layer 1's
    score slot stay at 0 ms: nothing else leaves them empty)."""
    c.pb200_xlinear_set_profile(h, 1)
    c.pb200_xlinear_reset_profile(h)
    out = run()
    prof = (c_double * (2 * depth))()
    c.pb200_xlinear_get_profile(h, prof)
    c.pb200_xlinear_set_profile(h, 0)
    return out, prof[1] == 0.0 and prof[2] == 0.0


def _resident(c, h, X, beam, topk, pp=None):
    from pecos_b200.core import ScipyCompressedSparseAllocator, ScipyCsrF32

    cx = ScipyCsrF32.init_from(X)
    c.pb200_xlinear_resident_upload_csr(h, byref(cx))
    c.pb200_xlinear_resident_predict(h, beam, pp.encode() if pp else None, topk, 0)
    alloc = ScipyCompressedSparseAllocator()
    c.pb200_xlinear_resident_fetch(h, alloc.cfunc)
    return alloc.get()


def _ab(c, h, depth, run, what, mode_on=1, expect=True):
    c.pb200_xlinear_set_lookup(h, 7)
    base, used = _profile(c, h, depth, run)
    assert not used, f"{what}: kernel mode 7 must not run the prefix kernel"
    c.pb200_xlinear_set_lookup(h, mode_on)
    got, used = _profile(c, h, depth, run)
    c.pb200_xlinear_set_lookup(h, 1)
    assert used == expect, f"{what}: prefix kernel {'not ' if expect else ''}used"
    _same_bits(got, base, what)
    return got


def test_prefix_eurlex_shape(tmp_path, gpu_clib, have_ref):
    """eurlex-4k's tree (4 / 64 / 3,956, D = 5,000, beam 10): resident batch (prefix by default), host CSR path (sub-tiles at
    workspace offsets, prefix forced), the oracles, and 7 kernels per resident step."""
    from oracle import ref, restatement
    from pecos_b200.xlinear import XLinearModel

    folder, X, cfg = synth.build_workload("eurlex-4k", str(tmp_path / "e"), scale_queries=8000)
    m = XLinearModel.load(folder, is_predict_only=True)
    c = gpu_clib.clib_float32
    h = m.model.model_chain
    beam, topk = cfg["beam_size"], cfg["only_topk"]
    got = _ab(c, h, 3, lambda: _resident(c, h, X, beam, topk), "eurlex resident")
    _ab(c, h, 3, lambda: m.predict(X, beam_size=beam, only_topk=topk), "eurlex host csr", mode_on=5)
    oracles = [restatement.OracleXLinear(os.path.join(folder, "ranker"))]
    if have_ref:
        oracles.append(ref.RefXLinear(os.path.join(folder, "ranker")))
    for o in oracles:
        assert_csr_parity(got[:100], o.predict(X[:100], beam, "l3-hinge", topk), what=f"eurlex prefix vs {type(o).__name__}")
    for mode, want in ((1, 7), (7, 16)):
        c.pb200_xlinear_set_lookup(h, mode)
        _resident(c, h, X, beam, topk)
        n0 = int(c.pb200_xlinear_launches(h))
        c.pb200_xlinear_resident_predict(h, beam, None, topk, 0)
        assert int(c.pb200_xlinear_launches(h)) - n0 == want, f"kernel mode {mode}: launches per resident step"
    c.pb200_xlinear_set_lookup(h, 1)


@pytest.mark.parametrize("saturate", [False, True])  # True: saturated hinge, layer 0's order decided by position
def test_prefix_post_processors_and_query_rows(tmp_path, gpu_clib, saturate):
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    layers = random_tree(161, [8, 64, 512], 400, 24, bias=1.0, saturate=saturate)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=8)
    X = csr_with_empty_rows(synth.make_queries(162, 3000, 400, 48), [0, 7, 2999])
    # a row without hits (a feature no weight row holds), and rows that repeat a column index
    W0, W1 = layers[0][0].tocsr(), layers[1][0].tocsr()
    unused = np.nonzero((np.diff(W0.indptr) == 0) & (np.diff(W1.indptr) == 0))[0]
    X = X.tolil()
    if unused.size:
        X.rows[5], X.data[5] = [int(unused[0])], [1.0]
    X = X.tocsr().astype(np.float32)
    for r in (3, 11, 500):
        s, e = X.indptr[r], X.indptr[r + 1]
        if e - s >= 4:
            X.indices[s + 1] = X.indices[s]
            X.indices[s + 3] = X.indices[s + 2]
    X.has_sorted_indices = True
    m = XLinearModel.load(folder, is_predict_only=True)
    c = gpu_clib.clib_float32
    h = m.model.model_chain
    for pp in ("l3-hinge", "sigmoid", "log-l2-hinge", "noop"):
        _ab(c, h, 3, lambda: m.predict(X, beam_size=10, only_topk=8, post_processor=pp), f"{pp} saturate={saturate}", mode_on=5)
        _ab(c, h, 3, lambda: _resident(c, h, X, 10, 8, pp), f"{pp} resident saturate={saturate}", mode_on=5)


def test_prefix_not_eligible(tmp_path, gpu_clib):
    """A beam narrower than layer 0, unequal biases and a rearranged layer 1 keep the per-layer kernels."""
    from pecos_b200.xlinear import XLinearModel

    c = gpu_clib.clib_float32
    X = synth.make_queries(172, 2500, 300, 30)
    # beam 4 < layer 0's 8 nodes
    folder = str(tmp_path / "a")
    synth.save_xlinear_model(folder, random_tree(171, [8, 64, 512], 300, 20), bias=1.0, only_topk=6)
    m = XLinearModel.load(folder, is_predict_only=True)
    h = m.model.model_chain
    _ab(c, h, 3, lambda: m.predict(X, beam_size=4, only_topk=6), "narrow beam", mode_on=5, expect=False)
    _ab(c, h, 3, lambda: m.predict(X, beam_size=8, only_topk=6), "full beam", mode_on=5, expect=True)
    # layer 0 with another bias than layer 1
    folder = str(tmp_path / "b")
    synth.save_xlinear_model(folder, random_tree(173, [8, 64, 512], 300, 20), bias=1.0, only_topk=6)
    p = os.path.join(folder, "ranker", "0.model", "param.json")
    meta = json.load(open(p))
    meta["bias"] = 0.5
    json.dump(meta, open(p, "w"))
    m = XLinearModel.load(folder, is_predict_only=True)
    h = m.model.model_chain
    _ab(c, h, 3, lambda: m.predict(X, beam_size=10, only_topk=6), "unequal bias", mode_on=5, expect=False)
    # rearranged (permuted) layer 1
    folder = str(tmp_path / "c")
    synth.save_xlinear_model(folder, random_tree(174, [8, 64, 512], 300, 20, permute=True), bias=1.0, only_topk=6)
    m = XLinearModel.load(folder, is_predict_only=True)
    h = m.model.model_chain
    _ab(c, h, 3, lambda: m.predict(X, beam_size=10, only_topk=6), "rearranged", mode_on=5, expect=False)


def test_prefix_across_workspace_tiles(tmp_path, gpu_clib, monkeypatch):
    """PB200_WORKSPACE_MB=64 cuts the resident batch into tiles of ~8,700 rows: the prefix serves each tile at its workspace
    offset (mode 5), or only the large ones (mode 1: the short last tile keeps the per-layer kernels)."""
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, random_tree(181, [2, 4, 1800], 400, 24), bias=1.0, only_topk=10)
    X = synth.make_queries(182, 20000, 400, 24)
    monkeypatch.setenv("PB200_WORKSPACE_MB", "64")
    m = XLinearModel.load(folder, is_predict_only=True)
    c = gpu_clib.clib_float32
    h = m.model.model_chain
    _ab(c, h, 3, lambda: _resident(c, h, X, 10, 10), "tiles forced", mode_on=5)
    c.pb200_xlinear_set_lookup(h, 7)
    base = _resident(c, h, X, 10, 10)
    c.pb200_xlinear_set_lookup(h, 1)
    _same_bits(_resident(c, h, X, 10, 10), base, "tiles default")
