"""The INTEGRATION.md overlay exercised END TO END on a GPU box.

The reference's Python package does not exist on the GPU box, so `pecos.core.clib` is played by a stand-in with the same two
attributes the overlay touches (`clib_float32`: a ctypes handle of the REFERENCE library oracle/_ref with the reference's
prototypes; `ann_hnsw_fn_dict`).  After `pecos_b200.integration.overlay(stand_in)`:
  * loading / predicting through the stand-in's function pointers runs on the GPU (handles are pecos_b200 handles) and returns
    the oracle's results,
  * symbols that are not served (HNSW train, ...) still run in the reference library, and the handles they create are forwarded
    back to it (pb200_hnsw_set_foreign).
tests/test_overlay_cpu.py checks the same overlay against the real reference Python package (binding only, no GPU there)."""
import ctypes
import gc
import json
import os

import numpy as np
import pytest

from pecos_b200 import synth

from .util import assert_csr_parity, random_tree

pytestmark = pytest.mark.gpu


def _run_through_the_overlay(tmp_path, gpu_clib, ref, restatement, folder, X, want):
    m = ref.RefXLinear(os.path.join(folder, "ranker"))
    assert gpu_clib.clib_float32.pb200_xlinear_replicas(m.h) == 1, "the handle must come from the CUDA library"
    assert_csr_parity(m.predict(X, 8, None, 5), want, what="overlaid c_xlinear_predict_csr_f32")
    assert_csr_parity(m.predict(X.toarray(), 8, None, 5), want, what="overlaid c_xlinear_predict_drm_f32")
    # compile (overlaid: this library's host-only writer of the reference's mmap format), load + predict through the overlay
    mm = str(tmp_path / "mm")
    os.makedirs(mm)
    ref.compile_mmap_model(os.path.join(folder, "ranker"), os.path.join(mm, "ranker"))
    m2 = ref.RefXLinear(os.path.join(mm, "ranker"), is_mmap=True)
    assert gpu_clib.clib_float32.pb200_xlinear_replicas(m2.h) == 1
    assert_csr_parity(m2.predict(X, 8, None, 5), want, what="reference-compiled mmap model through the overlay")
    # HNSW: train + save in the reference (not swapped), load + search through the overlay
    rng = np.random.default_rng(5)
    B = rng.standard_normal((800, 48)).astype(np.float32)
    Q = rng.standard_normal((40, 48)).astype(np.float32)
    idx = str(tmp_path / "idx")
    trained = ref.RefHNSW.train(B, M=8, efC=40, metric="l2", threads=1)
    trained.save(os.path.join(idx, "c_model"))
    json.dump({"model": "HNSW", "data_type": "drm", "metric_type": "l2", "num_item": 800, "feat_dim": 48}, open(os.path.join(idx, "param.json"), "w"))
    loaded = ref.RefHNSW.load(os.path.join(idx, "c_model"), "l2")  # overlaid load -> CUDA handle
    assert gpu_clib.clib_float32.pb200_hnsw_replicas(loaded.h) == 1
    gi, gd = loaded.predict(Q, 60, 10, threads=1)
    oi, od = restatement.OracleHNSW(idx, isa=0).predict(Q, 60, 10)
    assert np.array_equal(gi, oi) and np.array_equal(gd.view(np.uint32), od.view(np.uint32))
    # the TRAINED index is a reference handle: predict / searchers / destruct on it are forwarded to the reference library
    ti, td = trained.predict(Q, 60, 10, threads=1)
    assert np.array_equal(ti, oi)
    # save of an index loaded HERE = copy of the files it was loaded from; the copy loads and searches identically
    loaded.save(os.path.join(str(tmp_path / "idx2"), "c_model"))
    again = ref.RefHNSW.load(os.path.join(str(tmp_path / "idx2"), "c_model"), "l2")
    ai, ad = again.predict(Q, 60, 10, threads=1)
    assert np.array_equal(ai, oi) and np.array_equal(ad.view(np.uint32), od.view(np.uint32))


def test_overlay_end_to_end_on_a_stand_in_corelib(tmp_path, gpu_clib, have_ref, monkeypatch):
    if not have_ref:
        pytest.skip("needs the reference library (oracle/_ref) as the stand-in corelib the overlay re-points")
    import oracle
    from oracle import ref, restatement
    from pecos_b200 import integration

    class StandIn(object):
        pass

    stand_in = StandIn()
    stand_in.clib_float32 = ref.bind(ctypes.CDLL(oracle.REF_LIB))  # a fresh handle: the overlay mutates it
    stand_in.ann_hnsw_fn_dict = {}
    for metric in ("ip", "l2"):
        sfx = f"drm_{metric}_f32"
        stand_in.ann_hnsw_fn_dict[("drm", metric)] = {slot: getattr(stand_in.clib_float32, f"c_ann_hnsw_{slot}_{sfx}")
                                                      for slot in ("train", "load", "save", "destruct", "searchers_create",
                                                                   "searchers_destruct", "predict")}
    swapped = integration.overlay(stand_in)
    assert "c_xlinear_predict_csr_f32" in swapped and "c_ann_hnsw_predict_drm_ip_f32" in swapped
    assert "c_ann_hnsw_train_drm_l2_f32" not in swapped and "c_xlinear_compile_mmap_model" in swapped

    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, random_tree(411, [5, 30, 300], 200, 20, bias=1.0, permute=True), bias=1.0, only_topk=6)
    X = synth.make_queries(412, 200, 200, 30)
    want = restatement.OracleXLinear(os.path.join(folder, "ranker")).predict(X, 8, None, 5)
    monkeypatch.setattr(ref, "_lib", stand_in.clib_float32)  # drive the stand-in through the reference-style wrappers
    try:
        _run_through_the_overlay(tmp_path, gpu_clib, ref, restatement, folder, X, want)
    finally:
        gc.collect()  # handles created through the overlay are released while the overlay is still in place
