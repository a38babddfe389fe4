"""CPU tests of HNSW index sharding: the shard builder's manifest and files (pecos_b200/hnsw_build.py build_hnsw_shards on
device="cpu", tiny inputs), searches of every shard in the restatement and the reference library, and the exchange protocol
over torch.distributed with gloo at world size 2.  The GPU engine path is tests/test_hnsw_shard_gpu.py."""
import json
import os
import socket

import numpy as np
import pytest

from .hnsw_shard_util import hnsw_result_counts, hnsw_rows, hnsw_shard_records, merge_hnsw_shards_numpy
from .util import merge_shards_numpy

BUILD = dict(M=4, efC=16, device="cpu")


def _read(path):
    with open(path, "rb") as f:
        return f.read()


@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("world", [1, 3])
def test_shard_manifest_ranges_and_files(tmp_path, built, sparse, world):
    from pecos_b200.distributed import split_rows_by_nnz
    from pecos_b200.hnsw_build import build_hnsw_index, build_hnsw_shards

    X = hnsw_rows(1, 61, 24, sparse)
    folder = str(tmp_path / "s")
    out = build_hnsw_shards(X, folder, world, seed=5, metric="l2", pred_kwargs={"efS": 30}, **BUILD)
    man = json.load(open(os.path.join(folder, "shards.json")))
    assert man == out["manifest"]
    rb = man["row_begin"]
    assert len(rb) == world + 1 and rb[0] == 0 and rb[-1] == 61 and all(rb[r] < rb[r + 1] for r in range(world))
    if sparse:
        assert rb == split_rows_by_nnz(X.indptr, world)
    else:
        assert rb == [61 * r // world for r in range(world + 1)]
    assert man["world"] == world and man["num_item"] == 61 and man["feat_dim"] == 24
    assert man["data_type"] == ("csr" if sparse else "drm") and man["metric_type"] == "l2"
    assert man["seeds"] == [5 + r for r in range(world)] and man["pred_kwargs"] == {"efS": 30, "topk": 10, "threads": 1}
    for r in range(world):
        param = json.load(open(os.path.join(folder, f"shard-{r}", "param.json")))
        assert param["num_item"] == rb[r + 1] - rb[r] and param["pred_kwargs"] == man["pred_kwargs"]
    # shard r is build_hnsw_index of its rows with seed + r, byte for byte
    r = world - 1
    build_hnsw_index(X[rb[r]:rb[r + 1]], str(tmp_path / "one"), seed=5 + r, metric="l2", pred_kwargs={"efS": 30}, **BUILD)
    for name in ("c_model/index.mmap_store", "c_model/config.json", "param.json"):
        assert _read(os.path.join(folder, f"shard-{r}", name)) == _read(str(tmp_path / "one" / name)), name
    # one rank's call builds only its shard and writes the same manifest
    part = str(tmp_path / "part")
    build_hnsw_shards(X, part, world, ranks=[r], seed=5, metric="l2", pred_kwargs={"efS": 30}, **BUILD)
    assert sorted(os.listdir(part)) == sorted(["shards.json", f"shard-{r}"])
    assert _read(os.path.join(part, "shards.json")) == _read(os.path.join(folder, "shards.json"))


def test_shard_builder_rejects_empty_shards(tmp_path, built):
    from pecos_b200.hnsw_build import build_hnsw_shards

    with pytest.raises(ValueError, match="non-empty shards"):
        build_hnsw_shards(hnsw_rows(2, 3, 8, False), str(tmp_path / "s"), 4, **BUILD)
    with pytest.raises(ValueError, match="outside"):
        build_hnsw_shards(hnsw_rows(2, 30, 8, False), str(tmp_path / "s"), 2, ranks=[2], **BUILD)


@pytest.mark.parametrize("sparse,metric", [(False, "ip"), (False, "l2"), (True, "ip"), (True, "l2")])
def test_every_shard_searches_identically_in_restatement_and_reference(tmp_path, built, have_ref, sparse, metric):
    from oracle import restatement

    from pecos_b200.hnsw_build import build_hnsw_shards

    X, Q = hnsw_rows(3, 150, 32, sparse), hnsw_rows(4, 40, 32, sparse)
    folder = str(tmp_path / "s")
    rb = build_hnsw_shards(X, folder, 3, seed=7, metric=metric, **BUILD)["manifest"]["row_begin"]
    idx, dist = [], []
    for r in range(3):
        o = restatement.OracleHNSW(os.path.join(folder, f"shard-{r}"), isa=0)
        assert o.num_node == rb[r + 1] - rb[r]
        oi, od = o.predict(Q, 40, 10)
        if have_ref:
            from oracle import ref

            h = ref.RefHNSW.load(os.path.join(folder, f"shard-{r}", "c_model"), metric, data_type="csr" if sparse else "drm")
            ri, rd = h.predict(Q, 40, 10)
            assert np.array_equal(ri, oi) and np.array_equal(rd.view(np.uint32), od.view(np.uint32)), f"shard {r}"
        idx.append(oi)
        dist.append(od)
    # the merge of the per-shard lists: sorted by distance, ids within each shard's range
    m_ids, m_d = merge_hnsw_shards_numpy(np.stack(idx), np.stack(dist), rb, 10)
    assert np.all(np.diff(m_d, axis=1) >= 0) and m_ids.max() < rb[-1]


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
        man = json.load(open(os.path.join(folder, "shards.json")))
        rb, topk = man["row_begin"], 10
        Q = hnsw_rows(12, 50, 16, False)
        res = [restatement.OracleHNSW(os.path.join(folder, f"shard-{r}"), isa=0).predict(Q, 30, topk) for r in range(world)]
        li, ld = res[rank]
        keys, ids, vals = hnsw_shard_records(li, ld, hnsw_result_counts(li, ld), rank, rb[rank], topk)
        g = [comm.all_gather(torch.from_numpy(a)).numpy() for a in (keys.view(np.int64), ids.astype(np.int64), vals)]
        assert g[0].shape == (world, Q.shape[0], topk)
        assert np.array_equal(g[1][rank], ids)                # own slice sits at index `rank`
        g_keys = g[0].view(np.uint64)
        m_ids, m_vals, _ = merge_shards_numpy(g_keys, g[1].astype(np.uint32), g[2], (g_keys != 0).sum(2), topk)
        w_ids, w_vals = merge_hnsw_shards_numpy(np.stack([r[0] for r in res]), np.stack([r[1] for r in res]), rb, topk)
        assert np.array_equal(m_ids, w_ids) and np.array_equal(m_vals.view(np.uint32), w_vals.view(np.uint32))
        open(os.path.join(out_dir, f"ok{rank}"), "w").write("ok")
    finally:
        dist.destroy_process_group()


def test_hnsw_shard_exchange_protocol_gloo_world2(tmp_path, built):
    """Per-rank records by the key rule -> ONE all_gather -> merge == the host merge of all shards' searches."""
    import torch.multiprocessing as mp

    from pecos_b200.hnsw_build import build_hnsw_shards

    folder = str(tmp_path / "s")
    build_hnsw_shards(hnsw_rows(11, 200, 16, False), folder, 2, seed=3, **BUILD)
    out_dir = str(tmp_path / "out")
    os.makedirs(out_dir)
    mp.spawn(_worker, args=(2, _free_port(), folder, out_dir), nprocs=2, join=True)
    assert all(os.path.exists(os.path.join(out_dir, f"ok{r}")) for r in range(2))
