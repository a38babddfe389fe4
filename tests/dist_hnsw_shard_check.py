#!/usr/bin/env python
"""Multi-process check of HNSW index sharding over NCCL (not collected by pytest; launch with torchrun on >= 2 GPUs):

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 tests/dist_hnsw_shard_check.py

Every rank builds and loads its own shard (build_hnsw_shards with ranks=[rank]), all ranks search the same batch through
ShardedHNSW (ONE NCCL all-gather of the per-rank top-k), and rank 0 compares the result with the host merge of the per-shard
HNSW.predict results (must be bit-identical).  Prints one JSON line with timings."""
import json
import os
import shutil
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def main():
    import torch
    import torch.distributed as dist

    from pecos_b200 import core
    from pecos_b200.distributed import ShardedHNSW
    from pecos_b200.hnsw import HNSW
    from pecos_b200.hnsw_build import build_hnsw_shards
    from tests.hnsw_shard_util import hnsw_rows, merge_hnsw_shards_numpy

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    lib = core.get_clib()
    lib.set_device(local)
    folder = os.path.join(tempfile.gettempdir(), f"pb200_hnsw_shard_check_w{world}")
    X, Q = hnsw_rows(5, 50_000, 128, False), hnsw_rows(6, 5_000, 128, False)
    build_hnsw_shards(X, folder, world, ranks=[rank], seed=0, M=16, efC=100, device=f"cuda:{local}")
    dist.barrier()
    sharded = ShardedHNSW.load(folder, device=local)
    pp = HNSW.PredParams(efS=100, topk=10)
    got = sharded.predict(Q, pp, ret_csr=False)
    t0 = time.perf_counter()
    for _ in range(5):
        got = sharded.predict(Q, pp, ret_csr=False)
    dt = (time.perf_counter() - t0) / 5
    ok = True
    if rank == 0:
        rb = sharded.row_begin
        per = [HNSW.load(os.path.join(folder, f"shard-{r}")).predict(Q, pp, ret_csr=False) for r in range(world)]
        w_ids, w_d = merge_hnsw_shards_numpy(np.stack([p[0] for p in per]), np.stack([p[1] for p in per]), rb, 10)
        ok = np.array_equal(got[0], w_ids) and np.array_equal(got[1].view(np.uint32), w_d.view(np.uint32))
        print(json.dumps({"check": "hnsw_shard_nccl", "world": world, "bit_identical": bool(ok), "row_begin": rb,
                          "queries": int(Q.shape[0]), "exchange_bytes": sharded.last_exchange_bytes,
                          "e2e_ms_per_call": 1e3 * dt, "queries_per_s": Q.shape[0] / dt, "last_phase_ms": sharded.last_phase_ms}))
    dist.barrier()
    if rank == 0:
        shutil.rmtree(folder, ignore_errors=True)
    dist.destroy_process_group()
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
