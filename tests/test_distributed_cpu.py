"""CPU tests of the N>1 host logic: row/shard partitioning and the index-sharding exchange protocol over
``torch.distributed`` with the gloo backend, world_size 2 (the GPU path uses the same code with NCCL)."""
import os
import socket

import numpy as np
import pytest

from pecos_b200 import synth
from pecos_b200.distributed import split_rows_by_nnz

from .util import merge_shards_numpy, random_tree


def test_split_rows_by_nnz_balances_and_covers():
    X = synth.make_queries(3, 1000, 500, 20)
    X.data[:] = 1
    for world in (1, 2, 3, 8):
        b = split_rows_by_nnz(X.indptr, world)
        assert b[0] == 0 and b[-1] == 1000 and len(b) == world + 1 and all(b[i] <= b[i + 1] for i in range(world))
        nnz = np.diff(np.asarray(X.indptr)[b])
        assert nnz.max() - nnz.min() <= 2 * 20
    ragged = np.concatenate([[0], np.cumsum(np.r_[np.full(10, 1000), np.full(990, 1)])])
    b = split_rows_by_nnz(ragged, 4)
    assert b[-1] == 1000 and b[1] <= 4  # the heavy rows are spread, not piled on rank 0


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, folder, out_dir):
    import torch
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from oracle import restatement
        from pecos_b200.distributed import _TorchComm

        comm = _TorchComm()
        assert (comm.rank, comm.world) == (rank, world)
        X = synth.make_queries(5, 40, 200, 25)
        o = restatement.OracleXLinear(os.path.join(folder, "ranker"))
        k, beam = 7, 6
        full = o.predict(X, beam, None, 10_000)   # every candidate of the final layer, in rank order
        want = o.predict(X, beam, None, k)
        n_labels = full.shape[1]
        owner = (np.arange(n_labels) * world) // n_labels  # contiguous label ranges per rank (== leaf chunk ranges)
        keys = np.zeros((X.shape[0], k), dtype=np.int64)
        ids = np.zeros((X.shape[0], k), dtype=np.int32)
        vals = np.zeros((X.shape[0], k), dtype=np.float32)
        cnt = np.zeros(X.shape[0], dtype=np.int32)
        for q in range(X.shape[0]):
            lab = full.indices[full.indptr[q]:full.indptr[q + 1]]
            val = full.data[full.indptr[q]:full.indptr[q + 1]]
            mine = np.nonzero(owner[lab] == rank)[0][:k]     # local top-k: the best k owned candidates, order kept
            cnt[q] = mine.size
            ids[q, :mine.size] = lab[mine]
            vals[q, :mine.size] = val[mine]
            keys[q, :mine.size] = 1_000_000 - mine           # any strictly decreasing function of the global rank
        g = [comm.all_gather(torch.from_numpy(a)).numpy() for a in (keys, ids, vals, cnt)]
        assert g[0].shape == (world, X.shape[0], k) and g[3].shape == (world, X.shape[0])
        assert np.array_equal(g[1][rank], ids)               # own slice sits at index `rank`
        m_ids, m_vals, m_cnt = merge_shards_numpy(g[0].view(np.uint64), g[1], g[2], g[3], k)
        for q in range(X.shape[0]):
            w_lab = want.indices[want.indptr[q]:want.indptr[q + 1]]
            assert m_cnt[q] == w_lab.size
            assert np.array_equal(m_ids[q, :m_cnt[q]], w_lab)
            assert np.array_equal(m_vals[q, :m_cnt[q]], want.data[want.indptr[q]:want.indptr[q + 1]])
        open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    finally:
        dist.destroy_process_group()


def test_index_shard_exchange_protocol_gloo_world2(tmp_path, built):
    """Local top-k lists -> ONE all_gather -> merge == unsharded top-k (ids, ranks and score bits)."""
    import torch.multiprocessing as mp

    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, random_tree(13, [4, 20, 180], 200, 15, bias=1.0), bias=1.0, only_topk=6)
    out_dir = str(tmp_path / "out")
    os.makedirs(out_dir)
    world = 2
    mp.spawn(_worker, args=(world, _free_port(), folder, out_dir), nprocs=world, join=True)
    assert all(os.path.exists(os.path.join(out_dir, f"ok{r}")) for r in range(world))


def test_leaf_shard_ranges_cover_all_chunks(clib, tmp_path):
    """Host-side ownership split: contiguous, disjoint, complete, balanced by bytes (checked through the shard loader's
    reported ranges on the GPU; here only the pure function on synthetic weights via numpy re-implementation)."""
    w = np.r_[np.full(10, 1000), np.full(90, 10)].astype(np.int64)
    total = int((w + 1).sum())
    for world in (2, 3, 8):
        begin = [0]
        run, r = 0, 1
        for i, x in enumerate(w):
            run += int(x) + 1
            while r < world and run * world >= r * total:
                begin.append(i + 1)
                r += 1
        while len(begin) < world:
            begin.append(len(w))
        begin.append(len(w))
        assert begin[0] == 0 and begin[-1] == len(w) and all(begin[i] <= begin[i + 1] for i in range(world))
