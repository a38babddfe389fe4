"""GPU tests of leaf-layer index sharding (BASELINE.json configs[4]): several shard handles on ONE GPU emulate the ranks,
torch.stack emulates the all-gather; the merged result must be bit-identical to the unsharded prediction.
The real multi-process NCCL run is tests/dist_index_shard_check.py (launched with torchrun on >= 2 GPUs)."""
import os
from ctypes import byref, c_uint32, c_void_p

import numpy as np
import pytest

from pecos_b200 import synth

from .util import assert_csr_parity, random_tree

pytestmark = pytest.mark.gpu


def _sharded_predict(clib, ranker, X, world, beam, topk, pp=None):
    """The production exchange: every rank's local top-k as ONE buffer of 16-byte {key, id, value} records (key == 0: empty),
    ONE all-gather (emulated by torch.stack), merge of the gathered records.  Also returns the shard ranges and the number of
    local records (non-zero keys) over all ranks."""
    import torch

    from pecos_b200.core import ScipyCompressedSparseAllocator, ScipyCsrF32

    c = clib.clib_float32
    dev = torch.device("cuda", 0)
    handles = [c_void_p(c.pb200_xlinear_load_sharded(ranker.encode(), 2, r, world)) for r in range(world)]
    try:
        ranges = []
        for h in handles:
            out = (c_uint32 * 4)()
            c.pb200_xlinear_get_shard(h, out)
            ranges.append((int(out[2]), int(out[3])))
        assert ranges[0][0] == 0 and all(ranges[i][1] == ranges[i + 1][0] for i in range(world - 1))
        rows = X.shape[0]
        cx = ScipyCsrF32.init_from(X)
        recs, stride = [], None
        for h in handles:
            rec = torch.zeros((rows, topk, 2), dtype=torch.int64, device=dev)
            torch.cuda.synchronize()
            s = c.pb200_xlinear_sharded_local_csr_packed(h, byref(cx), beam, pp.encode() if pp else None, topk, topk, rec.data_ptr())
            assert stride in (None, s)
            stride = s
            recs.append(rec.view(-1)[: rows * s * 2].view(rows, s, 2))
        g = torch.stack(recs).contiguous()
        torch.cuda.synchronize()
        alloc = ScipyCompressedSparseAllocator()
        c.pb200_xlinear_sharded_merge_packed(handles[0], world, rows, stride, topk, g.data_ptr(), alloc.cfunc)
        return alloc.get(), ranges, int((g[..., 0] != 0).sum().item())
    finally:
        for h in handles:
            c.c_xlinear_destruct_model(h)


@pytest.mark.parametrize("world", [2, 3, 8])
def test_packed_index_sharded_prediction_is_bit_identical(tmp_path, gpu_clib, world):
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    layers = random_tree(91, [5, 40, 640], 400, 30, bias=1.0, permute=True)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=9)
    X = synth.make_queries(92, 120, 400, 40)
    whole = XLinearModel.load(folder, is_predict_only=True)
    for beam, topk, pp in [(6, 10, None), (3, 4, "noop"), (12, 10, "log-l2-hinge")]:
        want = whole.predict(X, beam_size=beam, only_topk=topk, post_processor=pp) if pp else whole.predict(X, beam_size=beam, only_topk=topk)
        got, ranges, n_local = _sharded_predict(gpu_clib, os.path.join(folder, "ranker"), X, world, beam, topk, pp)
        assert_csr_parity(got, want, rtol=0.0, what=f"world={world} beam={beam} topk={topk} pp={pp}")
        assert n_local >= want.nnz  # the union of the local lists covers the global top-k


def test_packed_exchange_saturated_ties_across_shards(tmp_path, gpu_clib):
    """All-tie scores: only the embedded global position can order candidates that live on different GPUs."""
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    layers = random_tree(93, [6, 48, 600], 200, 40, bias=1.0, permute=True, saturate=True)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=10)
    X = synth.make_queries(94, 64, 200, 50)
    want = XLinearModel.load(folder, is_predict_only=True).predict(X, beam_size=10, only_topk=10)
    assert np.mean(want.data == 1.0) > 0.2
    got, _, _ = _sharded_predict(gpu_clib, os.path.join(folder, "ranker"), X, 4, 10, 10)
    assert_csr_parity(got, want, rtol=0.0, what="saturated, world=4")


@pytest.mark.parametrize("world", [2, 8])
def test_packed_single_allgather_exchange_is_bit_identical(tmp_path, gpu_clib, world):
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    layers = random_tree(321, [8, 64, 900], 400, 30, bias=1.0, saturate=(world == 8))  # world 8: saturated hinge => ties decide
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=12)
    X = synth.make_queries(322, 333, 400, 40)
    want = XLinearModel.load(folder, is_predict_only=True).predict(X, beam_size=9, only_topk=12)
    got, _, _ = _sharded_predict(gpu_clib, os.path.join(folder, "ranker"), X, world, 9, 12)
    assert_csr_parity(got, want, rtol=0.0, what=f"packed exchange, world {world}")
