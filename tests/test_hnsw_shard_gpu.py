"""GPU tests of HNSW index sharding (pecos_b200.distributed.ShardedHNSW over shards written by build_hnsw_shards).  Several shard
handles on ONE GPU emulate the ranks and torch.stack emulates the all-gather.  The merged result must equal, bit for bit, the
numpy merge of the per-shard HNSW.predict results (merge_hnsw_shards_numpy in tests/hnsw_shard_util.py).  The real
multi-process NCCL run is tests/dist_hnsw_shard_check.py (launched with torchrun on >= 2 GPUs)."""
import json
import os

import numpy as np
import pytest

from .hnsw_shard_util import hnsw_result_counts, hnsw_rows, hnsw_shard_records, merge_hnsw_shards_numpy

pytestmark = pytest.mark.gpu


class _StackComm(object):
    """Rank `rank` of a `world` emulated on one GPU: all_gather keeps the local buffer (`sent`) and stacks it with the other
    ranks' buffers in `parts` (all-empty records where a part is not known yet)."""

    def __init__(self, rank, world, parts=None):
        self.rank, self.world, self.parts, self.sent = rank, world, parts, None

    def all_gather(self, local):
        import torch

        self.sent = local.clone()
        parts = self.parts or [torch.zeros_like(local)] * self.world
        return torch.stack([local if r == self.rank else parts[r] for r in range(self.world)]).contiguous()


def _records(rec):
    """[rows][topk] records (int64 pairs) -> keys u64, ids u32, distance bits u32."""
    a = rec.cpu().numpy()
    pair = np.ascontiguousarray(a[..., 1]).view(np.uint32).reshape(a.shape[0], a.shape[1], 2)
    return np.ascontiguousarray(a[..., 0]).view(np.uint64), pair[..., 0], pair[..., 1]


def _bits_equal(got, want, what):
    (gi, gd), (wi, wd) = got, want
    assert gi.shape == wi.shape, what
    bad = np.nonzero((gi != wi).any(1) | (gd.view(np.uint32) != wd.view(np.uint32)).any(1))[0]
    assert bad.size == 0, f"{what}: {bad.size} rows differ; first {bad[0]}: got {gi[bad[0]]} {gd[bad[0]]} want {wi[bad[0]]} {wd[bad[0]]}"


def _sharded_predict(folder, X, efS, topk, check_records=True):
    """Every rank's ShardedHNSW.predict with the all-gather emulated; returns rank 0's result (every rank's must be equal)
    and the expected numpy merge of the per-shard HNSW.predict results."""
    from pecos_b200.distributed import ShardedHNSW
    from pecos_b200.hnsw import HNSW

    man = json.load(open(os.path.join(folder, "shards.json")))
    world, rb = man["world"], man["row_begin"]
    pp = HNSW.PredParams(efS=efS, topk=topk)
    shards, sent, plain = [], [], []
    for r in range(world):
        s = ShardedHNSW.load(folder, comm=_StackComm(r, world))
        s.predict(X, pp, ret_csr=False)  # pass 1: this rank's records (the other ranks' slots are empty)
        shards.append(s)
        sent.append(s.comm.sent)
        plain.append(HNSW.load(os.path.join(folder, f"shard-{r}")).predict(X, pp, ret_csr=False))
        if check_records:  # the pack kernel against the key rule applied to the shard's own search
            li, ld = plain[-1]
            w_keys, w_ids, w_vals = hnsw_shard_records(li, ld, hnsw_result_counts(li, ld), r, rb[r], topk)
            g_keys, g_ids, g_bits = _records(s.comm.sent)
            assert np.array_equal(g_keys, w_keys) and np.array_equal(g_ids, w_ids), f"rank {r}: records differ"
            assert np.array_equal(g_bits, w_vals.view(np.uint32)), f"rank {r}: record distances differ"
    want = merge_hnsw_shards_numpy(np.stack([p[0] for p in plain]), np.stack([p[1] for p in plain]), rb, topk)
    got = None
    for r in sorted({0, world - 1}):
        shards[r].comm.parts = sent
        res = shards[r].predict(X, pp, ret_csr=False)
        assert shards[r].last_exchange_bytes == 16 * X.shape[0] * topk
        if got is None:
            got = res
        else:
            _bits_equal(res, got, f"rank {r} vs rank 0")
    return got, want, shards[0]


CASES = [(False, "ip"), (False, "l2"), (True, "ip"), (True, "l2")]


@pytest.mark.parametrize("world", [2, 3, 8])
@pytest.mark.parametrize("sparse,metric", CASES)
def test_sharded_search_equals_numpy_merge_of_shard_searches(tmp_path, gpu_clib, world, sparse, metric):
    from pecos_b200.hnsw_build import build_hnsw_shards

    X, Q = hnsw_rows(21, 800, 48, sparse), hnsw_rows(22, 150, 48, sparse)
    folder = str(tmp_path / "s")
    build_hnsw_shards(X, folder, world, seed=11, M=8, efC=40, metric=metric, device="cuda:0")
    for efS, topk in ((40, 10), (16, 24)):
        got, want, s0 = _sharded_predict(folder, Q, efS, topk)
        _bits_equal(got, want, f"world={world} {metric} sparse={sparse} efS={efS} topk={topk}")
    s0.comm.parts = None  # CSR form (rows x num_item, topk stored slots per row like HNSW.predict) of the same call
    csr = s0.predict(Q, s0.get_pred_params())
    idx, dist = s0.predict(Q, s0.get_pred_params(), ret_csr=False)
    assert csr.shape == (Q.shape[0], X.shape[0]) and np.array_equal(csr.indptr, np.arange(Q.shape[0] + 1) * idx.shape[1])
    assert np.array_equal(csr.indices, idx.ravel()) and np.array_equal(csr.data.view(np.uint32), dist.ravel().view(np.uint32))


@pytest.mark.parametrize("sparse,metric", [(False, "ip"), (True, "l2")])
def test_world1_shard_is_the_unsharded_index(tmp_path, gpu_clib, sparse, metric):
    from pecos_b200.distributed import ShardedHNSW
    from pecos_b200.hnsw import HNSW
    from pecos_b200.hnsw_build import build_hnsw_index, build_hnsw_shards

    X, Q = hnsw_rows(31, 1500, 40, sparse), hnsw_rows(32, 300, 40, sparse)
    kw = dict(M=8, efC=40, metric=metric, device="cuda:0")
    build_hnsw_shards(X, str(tmp_path / "s"), 1, seed=4, **kw)
    build_hnsw_index(X, str(tmp_path / "one"), seed=4, **kw)
    for name in ("c_model/index.mmap_store", "c_model/config.json", "param.json"):
        a = open(str(tmp_path / "s" / "shard-0" / name), "rb").read()
        assert a == open(str(tmp_path / "one" / name), "rb").read(), name
    s = ShardedHNSW.load(str(tmp_path / "s"), comm=_StackComm(0, 1))
    h = HNSW.load(str(tmp_path / "one"))
    for efS, topk in ((50, 10), (8, 20)):
        pp = HNSW.PredParams(efS=efS, topk=topk)
        _bits_equal(s.predict(Q, pp, ret_csr=False), h.predict(Q, pp, ret_csr=False), f"world 1 efS={efS} topk={topk}")
        a, b = s.predict(Q, pp), h.predict(Q, pp)
        assert a.shape == b.shape and np.array_equal(a.indices, b.indices) and np.array_equal(a.data.view(np.uint32), b.data.view(np.uint32))


def test_ties_across_shards_take_the_lower_rank_first(tmp_path, gpu_clib):
    """Two identical halves at world 2: every neighbour exists in both shards at the same distance."""
    from pecos_b200.hnsw_build import build_hnsw_shards

    B = hnsw_rows(41, 500, 32, False)
    folder = str(tmp_path / "s")
    build_hnsw_shards(np.vstack([B, B]), folder, 2, seed=2, M=8, efC=40, device="cuda:0")
    Q = hnsw_rows(42, 200, 32, False)
    (ids, dist), want, _ = _sharded_predict(folder, Q, 100, 10)
    _bits_equal((ids, dist), want, "tied halves")
    ties = 0
    for q in range(Q.shape[0]):
        for j in range(9):
            if dist[q, j] == dist[q, j + 1]:
                ties += 1
                assert ids[q, j] < 500 <= ids[q, j + 1] and ids[q, j + 1] - 500 == ids[q, j], (q, ids[q], dist[q])
    assert ties >= 4 * Q.shape[0]


@pytest.mark.parametrize("n,world,efS,topk", [(12, 3, 20, 10), (6, 2, 20, 10), (60, 3, 3, 10)])
def test_short_results_are_zero_filled_like_the_merge(tmp_path, gpu_clib, n, world, efS, topk):
    from pecos_b200.hnsw_build import build_hnsw_shards

    folder = str(tmp_path / "s")
    build_hnsw_shards(hnsw_rows(51, n, 16, False), folder, world, seed=1, M=4, efC=8, metric="l2", device="cuda:0")
    Q = hnsw_rows(52, 40, 16, False)
    got, want, _ = _sharded_predict(folder, Q, efS, topk)
    _bits_equal(got, want, f"n={n} world={world} efS={efS}")
    cnt = hnsw_result_counts(*want)
    assert np.all(cnt == min(n, topk))
    if n < topk:
        assert np.all(got[0][:, n:] == 0) and np.all(got[1][:, n:].view(np.uint32) == 0)


def test_rejections_happen_before_any_native_call(tmp_path, gpu_clib):
    import scipy.sparse as smat
    from ctypes import c_uint64

    from pecos_b200.distributed import ShardedHNSW
    from pecos_b200.hnsw import HNSW
    from pecos_b200.hnsw_build import build_hnsw_shards

    folder = str(tmp_path / "s")
    build_hnsw_shards(hnsw_rows(61, 100, 16, False), folder, 2, M=4, efC=8, device="cuda:0")
    with pytest.raises(ValueError, match="holds 2 shards"):
        ShardedHNSW.load(folder, comm=_StackComm(0, 3))
    s = ShardedHNSW.load(folder, comm=_StackComm(1, 2))

    def launches():
        out = (c_uint64 * 8)()
        gpu_clib.clib_float32.pb200_hnsw_get_info(s.index.model_ptr, out)
        return int(out[7])

    before = launches()
    Q = hnsw_rows(62, 5, 16, False)
    with pytest.raises(ValueError, match="merge capacity"):
        s.predict(Q, HNSW.PredParams(efS=600, topk=513))
    with pytest.raises(ValueError, match="csr queries cannot be searched"):
        s.predict(smat.csr_matrix(Q))
    with pytest.raises(ValueError, match="query dimension 15"):
        s.predict(Q[:, :15])
    assert launches() == before and s.comm.sent is None


def test_sharded_recall_is_at_the_unsharded_level(tmp_path, gpu_clib):
    from pecos_b200.hnsw import HNSW
    from pecos_b200.hnsw_build import build_hnsw_index, build_hnsw_shards

    X, Q = hnsw_rows(71, 20000, 64, False), hnsw_rows(72, 2000, 64, False)
    kw = dict(M=16, efC=100, metric="ip", device="cuda:0")
    build_hnsw_index(X, str(tmp_path / "one"), seed=0, **kw)
    build_hnsw_shards(X, str(tmp_path / "s"), 4, seed=0, **kw)
    exact = np.argsort(1.0 - Q @ X.T, axis=1, kind="stable")[:, :10]
    pp = HNSW.PredParams(efS=100, topk=10)

    def recall(idx):
        return float(np.mean([len(set(idx[i].tolist()) & set(exact[i].tolist())) / 10.0 for i in range(Q.shape[0])]))

    r_one = recall(HNSW.load(str(tmp_path / "one")).predict(Q, pp, ret_csr=False)[0])
    (ids, _), want, _ = _sharded_predict(str(tmp_path / "s"), Q, 100, 10, check_records=False)
    r_sharded = recall(ids)
    assert r_sharded >= r_one - 0.01, f"recall@10 sharded (world 4) {r_sharded:.4f} vs unsharded {r_one:.4f}"
    print(f"recall@10 efS=100: unsharded {r_one:.4f}, world 4 {r_sharded:.4f}")
