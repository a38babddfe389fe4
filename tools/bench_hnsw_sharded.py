#!/usr/bin/env python
"""Measures HNSW index sharding: one shard per rank (build_hnsw_shards, built in parallel), searched through ShardedHNSW with
ONE all-gather of the per-rank top-k, next to the unsharded index (world 1) of the same rows.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 tools/bench_hnsw_sharded.py [--out DIR]

(plain ``python tools/bench_hnsw_sharded.py`` runs world 1 only.)  Defaults: bench.py's hnsw-1m shape (1M x 768 unit rows, ip,
M 32, efC 100, 50,000 queries, efS 200, top-10), rows and queries generated as bench.py does for its dense HNSW workloads.
Indices are cached under --cache-dir by shape, world and seed.  Per world: warm ShardedHNSW.predict calls timed with host
clocks around device-synchronised work (split into local search, exchange and merge), queries/s, recall@10 against the exact
top-10, index bytes in HBM and build time per rank, exchange bytes.  Rank 0 prints one JSON line with the card's name and
power limit."""
import argparse
import ctypes
import datetime
import json
import os
import socket
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import HNSW_WORKLOADS  # noqa: E402
from tools.bench_hnsw_build import card, exact_top10, recall  # noqa: E402


class _SelfComm(object):
    """world 1 without a collective (the unsharded index searched through the same ShardedHNSW path)."""

    rank, world = 0, 1

    def all_gather(self, local):
        return local.unsqueeze(0)


def unit_rows(seed, n, d):
    """bench.py's dense HNSW rows: standard normal, row-normalised (seed 30: base rows, 31: rank 0's queries)."""
    X = np.random.default_rng(seed).standard_normal((n, d), dtype=np.float32)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    return X


def build_or_load(args, X, world, rank, local):
    """This rank's shard of the world-`world` layout in the cache; returns (folder, build seconds of this rank, recorded
    when it was built)."""
    from pecos_b200.hnsw_build import build_hnsw_shards

    folder = os.path.join(args.cache_dir, f"{args.N}x{args.d}-M{args.M}-efC{args.efC}-{args.metric}-w{world}-s{args.seed}")
    done = os.path.join(folder, f"built-{rank}.json")
    if os.path.exists(done) and os.path.exists(os.path.join(folder, "shards.json")):
        return folder, json.load(open(done))["build_s"]
    import torch

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    build_hnsw_shards(X, folder, world, ranks=[rank], device=f"cuda:{local}", seed=args.seed, M=args.M, efC=args.efC,
                      metric=args.metric, pred_kwargs={"efS": args.efS, "topk": args.topk})
    torch.cuda.synchronize()
    build_s = time.perf_counter() - t0
    with open(done, "w") as f:
        json.dump({"build_s": build_s}, f)
    return folder, build_s


def measure(args, sharded, Q, exact):
    from pecos_b200.hnsw import HNSW

    c = sharded._clib.clib_float32
    pp = HNSW.PredParams(efS=args.efS, topk=args.topk)
    for _ in range(args.warmup):
        sharded.predict(Q, pp, ret_csr=False)
    steps, phases = [], []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        idx, _ = sharded.predict(Q, pp, ret_csr=False)  # ends with the merged result on the host
        steps.append(time.perf_counter() - t0)
        phases.append(sharded.last_phase_ms)
    info = (ctypes.c_uint64 * 8)()
    c.pb200_hnsw_get_info(sharded.index.model_ptr, info)
    out = {"step_ms_median": 1e3 * float(np.median(steps)), "step_ms_min": 1e3 * float(np.min(steps)),
           "queries_per_s": Q.shape[0] / float(np.median(steps)),
           "phase_ms_median": {k: float(np.median([p[k] for p in phases])) for k in phases[0]},
           "exchange_bytes_per_rank": sharded.last_exchange_bytes, "index_bytes_this_rank": int(info[6])}
    if exact is not None:
        out["recall@10"] = recall(idx, exact)
    return out


def main():
    w = HNSW_WORKLOADS["hnsw-1m"]
    ap = argparse.ArgumentParser()
    ap.add_argument("--N", type=int, default=w["N"])
    ap.add_argument("--d", type=int, default=w["d"])
    ap.add_argument("--M", type=int, default=w["M"])
    ap.add_argument("--efC", type=int, default=w["efC"])
    ap.add_argument("--metric", default=w["metric"], choices=["ip", "l2"])
    ap.add_argument("--queries", type=int, default=w["Q"])
    ap.add_argument("--efS", type=int, default=w["efS"])
    ap.add_argument("--topk", type=int, default=w["topk"])
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cache-dir", default=os.path.join(tempfile.gettempdir(), "pb200_hnsw_sharded"))
    ap.add_argument("--out", default=None, help="also write the JSON result into this directory")
    args = ap.parse_args()

    import torch
    import torch.distributed as dist

    if not torch.cuda.is_available():
        raise SystemExit("bench_hnsw_sharded: no CUDA device visible (this measurement runs on the GPU only)")
    if "RANK" not in os.environ:  # single process: a world-1 group, so both legs run the same code
        s = socket.socket()
        s.bind(("127.0.0.1", 0))
        os.environ.update(RANK="0", WORLD_SIZE="1", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(s.getsockname()[1]))
        s.close()
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    # builds of the unsharded index on rank 0 can take long while the other ranks wait at a barrier
    dist.init_process_group("nccl", device_id=torch.device("cuda", local), timeout=datetime.timedelta(hours=3))
    from pecos_b200 import core
    from pecos_b200.distributed import ShardedHNSW

    core.get_clib().set_device(local)
    os.makedirs(args.cache_dir, exist_ok=True)
    X = unit_rows(30, args.N, args.d)
    Q = unit_rows(31, args.queries, args.d)
    res = {"card": card() if rank == 0 else None, "N": args.N, "d": args.d, "M": args.M, "efC": args.efC, "metric": args.metric,
           "queries": args.queries, "efS": args.efS, "topk": args.topk, "world": world, "runs": {}}
    exact = exact_top10(X, Q, args.metric) if rank == 0 else None
    legs = [world] + ([1] if world > 1 else [])
    for leg in legs:
        if leg == 1 and rank != 0:
            dist.barrier()
            continue
        folder, build_s = build_or_load(args, X, leg, rank, local)
        if leg > 1:
            dist.barrier()  # every shard and the manifest are on disk
            sharded = ShardedHNSW.load(folder, device=local)
        else:
            sharded = ShardedHNSW.load(folder, comm=_SelfComm(), device=local)
        r = measure(args, sharded, Q, exact if rank == 0 else None)
        if leg > 1:
            per = torch.tensor([build_s, float(r["index_bytes_this_rank"])], dtype=torch.float64, device="cuda")
            g = [torch.zeros_like(per) for _ in range(world)]
            dist.all_gather(g, per)
            r["build_s_per_rank"] = [float(t[0]) for t in g]
            r["index_bytes_per_rank"] = [int(t[1]) for t in g]
        else:
            r["build_s_per_rank"] = [build_s]
            r["index_bytes_per_rank"] = [r["index_bytes_this_rank"]]
            if world > 1:
                dist.barrier()
        del r["index_bytes_this_rank"]
        r["row_begin"] = sharded.row_begin
        res["runs"][f"world{leg}"] = r
        del sharded
    if rank == 0:
        line = json.dumps(res)
        print(line)
        if args.out:
            os.makedirs(args.out, exist_ok=True)
            with open(os.path.join(args.out, f"bench_hnsw_sharded_w{world}.json"), "w") as f:
                f.write(line + "\n")
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
