"""GPU tests of the XR-Linear engine's tiled batch loop.

Every entry point runs once at the default device workspace (one tile) and once with PB200_WORKSPACE_MB at its 64 MiB floor,
which cuts the same call into several tiles.  Queries are scored independently of their tile, so label ids, row lengths
and score bits must be identical.  The engine's launch counter shows that the small budget really tiled the call."""
import os
from ctypes import byref, c_uint32, c_void_p

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .util import assert_csr_parity, random_tree

pytestmark = pytest.mark.gpu

ROWS, D, BEAM, TOPK = 5000, 300, 64, 10


@pytest.fixture(scope="module")
def tiling_model(tmp_path_factory):
    """64 parents over 16,384 labels (leaf chunks of 256 columns on average).  At beam 64 a query needs about 64 KiB of
    workspace, so the 64 MiB floor holds about 1,000 queries per tile, and 5,000 CSR queries take the upload schedule
    with two staging sets."""
    folder = str(tmp_path_factory.mktemp("tiling") / "m")
    layers = random_tree(501, [64, 16384], D, 20, bias=1.0)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=TOPK)
    X = synth.make_queries(502, ROWS, D, 30)
    sel = smat.random(ROWS, 16384, density=0.005, format="csr", dtype=np.float32, random_state=np.random.default_rng(503))
    sel.sort_indices()
    return folder, layers, X, sel


def _tiled_equals_untiled(monkeypatch, c, handles, call, what):
    """call() at the default workspace and at the 64 MiB floor: identical results, more launches at the floor."""
    def launches():
        return sum(c.pb200_xlinear_launches(h) for h in handles)

    monkeypatch.delenv("PB200_WORKSPACE_MB", raising=False)
    l0 = launches()
    want = call()
    l1 = launches()
    monkeypatch.setenv("PB200_WORKSPACE_MB", "64")
    try:
        got = call()
    finally:
        monkeypatch.delenv("PB200_WORKSPACE_MB", raising=False)
    l2 = launches()
    assert want.nnz > 0, what
    assert assert_csr_parity(got, want, rtol=0.0, what=what) == 1.0, f"{what}: score bits differ"
    if handles:
        assert l2 - l1 > l1 - l0, f"{what}: {l2 - l1} launches at the floor vs {l1 - l0} in one tile: the call was not tiled"


def test_hierarchical_entry_points_tile(tiling_model, gpu_clib, monkeypatch):
    from pecos_b200.core import ScipyCompressedSparseAllocator, ScipyCsrF32
    from pecos_b200.xlinear import XLinearModel

    folder, _, X, sel = tiling_model
    c = gpu_clib.clib_float32
    m = XLinearModel.load(folder, is_predict_only=True)
    h = m.model.model_chain
    Xd = np.ascontiguousarray(X.toarray())
    _tiled_equals_untiled(monkeypatch, c, [h], lambda: m.predict(X, beam_size=BEAM, only_topk=TOPK), "csr")
    _tiled_equals_untiled(monkeypatch, c, [h], lambda: m.predict(Xd, beam_size=BEAM, only_topk=TOPK), "dense")

    cx = ScipyCsrF32.init_from(X)
    c.pb200_xlinear_resident_upload_csr(h, byref(cx))

    def resident():
        c.pb200_xlinear_resident_predict(h, BEAM, None, TOPK, 0)
        alloc = ScipyCompressedSparseAllocator()
        c.pb200_xlinear_resident_fetch(h, alloc.cfunc)
        return alloc.get()

    _tiled_equals_untiled(monkeypatch, c, [h], resident, "resident")
    _tiled_equals_untiled(monkeypatch, c, [h], lambda: m.predict(X, selected_outputs_csr=sel), "selected outputs")


def test_single_layer_entry_points_tile(tmp_path, tiling_model, gpu_clib, monkeypatch):
    from oracle import ref  # the ctypes wrapper of the c_mlmodel_* calls only
    from pecos_b200.xlinear import MLModel

    folder, layers, X, sel = tiling_model
    c = gpu_clib.clib_float32
    (W0, C0), (W1, C1) = layers
    codes = MLModel(W0, C0, bias=1.0).predict(X, only_topk=BEAM, post_processor="l3-hinge")  # every parent of every query
    leaf = MLModel(W1, C1, bias=1.0)
    for cc in (None, codes):
        _tiled_equals_untiled(monkeypatch, c, [], lambda: leaf.predict(X, csr_codes=cc, only_topk=TOPK, post_processor="l3-hinge"),
                              f"single layer, codes={cc is not None}")
    mm = str(tmp_path / "leaf_mmap")
    ref.compile_mlmodel_mmap(os.path.join(folder, "ranker", "1.model"), mm, clib=c)
    g = ref.MLModelHandle(mm, clib=c)
    for cc in (None, codes):
        _tiled_equals_untiled(monkeypatch, c, [g.h], lambda: g.predict(X, cc, None, TOPK), f"mlmodel, codes={cc is not None}")
    _tiled_equals_untiled(monkeypatch, c, [g.h], lambda: g.predict_on_selected_outputs(X, sel, codes, None),
                          "mlmodel selected outputs with codes")


def test_index_sharded_run_tiles(tiling_model, gpu_clib, monkeypatch):
    """Emulated world of 2 on one GPU: both ranks' local top-k (packed records) and the merge."""
    import torch

    from pecos_b200.core import ScipyCompressedSparseAllocator, ScipyCsrF32

    folder, _, X, _ = tiling_model
    c = gpu_clib.clib_float32
    world = 2
    handles = [c_void_p(c.pb200_xlinear_load_sharded(os.path.join(folder, "ranker").encode(), 2, r, world)) for r in range(world)]
    try:
        out = (c_uint32 * 4)()
        c.pb200_xlinear_get_shard(handles[1], out)
        assert 0 < out[2] < out[3]
        cx = ScipyCsrF32.init_from(X)
        dev = torch.device("cuda", 0)

        def sharded():
            recs = []
            for h in handles:
                rec = torch.zeros((ROWS, TOPK, 2), dtype=torch.int64, device=dev)
                torch.cuda.synchronize()
                assert c.pb200_xlinear_sharded_local_csr_packed(h, byref(cx), BEAM, None, TOPK, TOPK, rec.data_ptr()) == TOPK
                recs.append(rec)
            g = torch.stack(recs).contiguous()
            torch.cuda.synchronize()
            alloc = ScipyCompressedSparseAllocator()
            c.pb200_xlinear_sharded_merge_packed(handles[0], world, ROWS, TOPK, TOPK, g.data_ptr(), alloc.cfunc)
            return alloc.get()

        _tiled_equals_untiled(monkeypatch, c, handles, sharded, "index sharded, world 2")
    finally:
        for h in handles:
            c.c_xlinear_destruct_model(h)


def test_resident_batch_survives_host_buffer_calls(tiling_model, gpu_clib):
    """The resident batch and its results have their own device buffers: host-buffer predict calls in between -- one larger
    in rows and non-zeros than the resident batch, so every staging buffer grows, and one smaller -- change neither what
    resident_fetch returns nor what the next resident_predict computes."""
    from pecos_b200.core import ScipyCompressedSparseAllocator, ScipyCsrF32
    from pecos_b200.xlinear import XLinearModel

    folder, _, X, _ = tiling_model
    c = gpu_clib.clib_float32
    m = XLinearModel.load(folder, is_predict_only=True)
    h = m.model.model_chain
    Xr = X[:2000]
    assert X.nnz > Xr.nnz
    cx = ScipyCsrF32.init_from(Xr)
    c.pb200_xlinear_resident_upload_csr(h, byref(cx))

    def fetch():
        alloc = ScipyCompressedSparseAllocator()
        c.pb200_xlinear_resident_fetch(h, alloc.cfunc)
        return alloc.get()

    c.pb200_xlinear_resident_predict(h, BEAM, None, TOPK, 0)
    first = fetch()
    assert first.nnz > 0
    assert assert_csr_parity(first, m.predict(Xr, beam_size=BEAM, only_topk=TOPK), rtol=0.0, what="resident") == 1.0
    m.predict(X, beam_size=BEAM, only_topk=TOPK)
    m.predict(X[:300], beam_size=BEAM, only_topk=TOPK)
    assert assert_csr_parity(fetch(), first, rtol=0.0, what="fetch after host-buffer calls") == 1.0
    c.pb200_xlinear_resident_predict(h, BEAM, None, TOPK, 0)
    assert assert_csr_parity(fetch(), first, rtol=0.0, what="resident_predict after host-buffer calls") == 1.0
