"""CPU checks behind tests/test_index_shard_limits_gpu.py: the host plan's result stride (pb200_xlinear_plan_stride) is the
last layer's k_cap, and ShardedXLinearModel.predict refuses a call whose world x stride exceeds the merge capacity of 1024
records per query, or queries that are not a float32 csr matrix with sorted indices, with a ValueError before any native
call.  The model below is backed by a host-only handle and a stub library whose native calls fail the test."""
import json
import os

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .test_xlinear_limits_gpu import _queries, _two_layer
from .util import random_tree


def _k_cap_chain(layouts, stored_topk, beam_size, only_topk):
    """The last layer's k_cap of XLinearEngine::make_plan_, from the host layout: b_prev = 1 at the root, then
    max(1, min(k, b_prev x c_max)) per layer, k = beam_size above the leaf and only_topk at it (0: the stored value)."""
    b_prev = 1
    for d, L in enumerate(layouts):
        local = only_topk if d + 1 == len(layouts) else beam_size
        k = local or stored_topk[d]
        b_prev = max(1, min(k, b_prev * max(L["c_max"], 1)))
    return b_prev


def _save(folder, layers, only_topk=10):
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=only_topk)
    return os.path.join(folder, "ranker")


@pytest.mark.parametrize("sizes,topk", [([5, 40, 640], 10), ([8, 64, 900], 12), ([3, 6, 60], 7), ([16], 4), ([4, 200], 300)])
def test_plan_stride_is_the_last_layers_k_cap(tmp_path, clib, sizes, topk):
    ranker = _save(str(tmp_path / "m"), random_tree(len(sizes) * 10 + topk, sizes, 120, 8, bias=1.0, permute=True), topk)
    layouts = clib.host_model_layout(ranker)
    stored = [json.load(open(os.path.join(ranker, f"{d}.model", "param.json")))["pred_kwargs"]["only_topk"]
              for d in range(len(sizes))]
    c = clib.clib_float32
    h = c.pb200_xlinear_host_load(ranker.encode(), 0)
    try:
        for beam in (0, 1, 2, 5, 40, 1 << 20):
            for k in (0, 1, 7, 64, 200, 5000, 1 << 30):
                want = _k_cap_chain(layouts, stored, beam, k)
                assert clib.xlinear_plan_stride(h, beam, k, host=True) == want, (sizes, beam, k)
    finally:
        c.pb200_xlinear_host_free(h)


class _NoNative(object):
    def __getattr__(self, name):
        raise AssertionError(f"the native call {name} was reached")


class _HostOnly(object):
    """The library calls ShardedXLinearModel makes: the host plan checks answer from the host-only handle, every native
    call fails the test."""

    def __init__(self, clib):
        self.clib = clib
        self.clib_float32 = _NoNative()

    def xlinear_check_plan(self, model, beam_size, only_topk):
        return self.clib.xlinear_check_plan(model, beam_size, only_topk, host=True)

    def xlinear_plan_stride(self, model, beam_size, only_topk):
        return self.clib.xlinear_plan_stride(model, beam_size, only_topk, host=True)

    def xlinear_destruct_model(self, model):
        pass


class _NoComm(object):
    def all_gather(self, local):
        raise AssertionError("the exchange was reached")


@pytest.fixture(scope="module")
def wide_leaf(tmp_path_factory, clib):
    """Layer 0: one chunk of 48 nodes; leaf: 48 chunks of 64 columns (beam 40: 2,560 candidates per leaf row)."""
    ranker = _save(str(tmp_path_factory.mktemp("wide") / "m"), _two_layer(721, [64] * 48, 500, 12))
    pp = [json.load(open(os.path.join(ranker, f"{d}.model", "param.json")))["pred_kwargs"] for d in range(2)]
    h = clib.clib_float32.pb200_xlinear_host_load(ranker.encode(), 0)
    yield h, pp
    clib.clib_float32.pb200_xlinear_host_free(h)


def _sharded(clib, wide_leaf, world):
    from pecos_b200.distributed import ShardedXLinearModel

    h, pp = wide_leaf
    return ShardedXLinearModel(h, 0, world, _NoComm(), _HostOnly(clib), pp)


@pytest.mark.parametrize("world,beam,topk,stride", [(5, 40, 205, 205), (8, 40, 129, 129), (3, 40, 400, 400),
                                                    (9, 2, 200, 128), (2, 40, 513, 513)])
def test_too_wide_sharded_topk_raises_before_any_native_call(clib, wide_leaf, world, beam, topk, stride):
    m = _sharded(clib, wide_leaf, world)
    X = _queries(1, 500, [10, 20])
    narrow = f" \\(stride {stride} of top-k {topk}: [^)]*\\)" if stride != topk else ""
    with pytest.raises(ValueError, match=f"world \\* top-k = {world * stride}{narrow} exceeds the merge capacity of 1024 "
                                         "records per query"):
        m.predict(X, beam_size=beam, only_topk=topk)


@pytest.mark.parametrize("world,beam,topk", [(2, 40, 512), (4, 40, 256), (8, 40, 128), (8, 2, 200), (1, 40, 1024)])
def test_sharded_topk_at_the_merge_capacity_goes_on_to_the_native_call(clib, wide_leaf, world, beam, topk):
    """world x stride = 1024 (at beam 2 the stride is 128, the candidates a leaf row holds, not the requested 200)."""
    m = _sharded(clib, wide_leaf, world)
    X = _queries(2, 500, [10, 20])
    with pytest.raises(AssertionError, match="native call"):
        m.predict(X, beam_size=beam, only_topk=topk)


def test_queries_are_checked_before_any_native_call(clib, wide_leaf):
    m = _sharded(clib, wide_leaf, 2)
    X = _queries(3, 500, [10, 20, 30])
    with pytest.raises(ValueError, match="csr queries only"):
        m.predict(np.ascontiguousarray(X.toarray()), beam_size=4, only_topk=10)
    U = X.copy()
    U.indices[:3] = U.indices[:3][::-1].copy()  # row 0 no longer sorted
    U.has_sorted_indices = False
    with pytest.raises(ValueError, match="Query matrix does not have sorted indices!"):
        m.predict(U, beam_size=4, only_topk=10)
    with pytest.raises(ValueError, match="is not float32"):
        m.predict(smat.csr_matrix(X, dtype=np.float64), beam_size=4, only_topk=10)
    with pytest.raises(AssertionError, match="native call"):  # and a valid call reaches the native side
        m.predict(X, beam_size=4, only_topk=10)
