#!/usr/bin/env python
"""Measures the GPU build of a sparse (csr) HNSW index: build time and its split by phase, the work the distance kernels did,
and the recall of the written index searched by the CUDA engine.

    python tools/bench_hnsw_build.py [--workload hnsw-sparse-100k | hnsw-rcv1] [--compare-reference] [--out DIR]

Base rows: bench.make_sparse_rows(30, N, d, nnz) of the workload's shape (bench.py's HNSW_WORKLOADS); queries:
make_sparse_rows(31, Q, d, nnz).  Recall@10 at efS in {50, 100, 200} against the exact top-10 computed on the GPU.
--compare-reference (needs oracle/_ref): also trains the same rows with the reference's HNSW.train on all host threads
(same M, efC) and reports its build time and recall on the same queries.  Prints one JSON line.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import HNSW_WORKLOADS, make_sparse_rows  # noqa: E402

EFS = (50, 100, 200)


def card():
    import torch

    out = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        out["power_limit_w"] = float(r.stdout.strip().splitlines()[0])
    except Exception as e:  # reported, not guessed
        out["power_limit_error"] = repr(e)
    return out


def exact_top10(X, Q, metric, tile=512):
    """Exact top-10 by the reference's distance order on the GPU.  Sparse X (csr): ip 1 - <q,x> and the reference's l2 -2<q,x>,
    both = descending dot.  Dense X (float32 array): ip 1 - <q,x> (descending dot), l2 |q - x|^2 (descending 2<q,x> - |x|^2)."""
    import scipy.sparse as smat
    import torch

    dev = torch.device("cuda", 0)
    sparse = smat.issparse(X)
    if sparse:
        Xt = torch.sparse_csr_tensor(torch.from_numpy(X.indptr.astype(np.int64)), torch.from_numpy(X.indices.astype(np.int64)),
                                     torch.from_numpy(X.data), size=X.shape).to(dev)
    else:
        Xt = torch.from_numpy(np.ascontiguousarray(X, dtype=np.float32)).to(dev)
        sq = (Xt * Xt).sum(1) if metric == "l2" else None
    out = np.empty((Q.shape[0], 10), dtype=np.int64)
    for q0 in range(0, Q.shape[0], tile):
        q1 = min(Q.shape[0], q0 + tile)
        if sparse:
            dot = (Xt @ torch.from_numpy(Q[q0:q1].toarray()).to(dev).T).T   # [tile, N]
        else:
            dot = torch.from_numpy(np.ascontiguousarray(Q[q0:q1], dtype=np.float32)).to(dev) @ Xt.T
            if sq is not None:
                dot = 2.0 * dot - sq
        out[q0:q1] = torch.topk(dot, 10, dim=1, largest=True, sorted=True).indices.cpu().numpy()
    return out


def recall(idx, exact):
    return float(np.mean([len(set(idx[i].tolist()) & set(exact[i].tolist())) / 10.0 for i in range(idx.shape[0])]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="hnsw-sparse-100k", choices=["hnsw-sparse-100k", "hnsw-rcv1"])
    ap.add_argument("--queries", type=int, default=10_000)
    ap.add_argument("--compare-reference", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON result into this directory")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("bench_hnsw_build: no CUDA device visible (this measurement runs on the GPU only)")
    from pecos_b200.hnsw import HNSW
    from pecos_b200.hnsw_build import build_hnsw_index

    cfg = HNSW_WORKLOADS[args.workload]
    N, D, nnz, M, efC, metric = cfg["N"], cfg["d"], cfg["nnz"], cfg["M"], cfg["efC"], cfg["metric"]
    res = {"workload": args.workload, "card": card(), "N": N, "D": D, "M": M, "efC": efC, "metric": metric}
    t0 = time.perf_counter()
    X = make_sparse_rows(30, N, D, nnz)
    Q = make_sparse_rows(31, args.queries, D, nnz)
    res["generate_s"] = time.perf_counter() - t0
    res["stored_entries_per_row"] = X.nnz / N

    with tempfile.TemporaryDirectory() as tmp:
        folder = os.path.join(tmp, "idx")
        build_hnsw_index(make_sparse_rows(30, 2000, D, nnz), os.path.join(tmp, "warm"), M=M, efC=efC, metric=metric)  # loads, JIT
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        stats = build_hnsw_index(X, folder, M=M, efC=efC, metric=metric, seed=0, device="cuda:0")
        torch.cuda.synchronize()
        res["build_s"] = time.perf_counter() - t0
        res["phase_ms"] = stats["phase_ms"]
        res["work"] = {"block_postings": stats["block_postings"], "candidate_row_entries": stats["candidate_entries"]}
        res["nodes_per_level"] = stats["nodes_per_level"]
        res["mean_degree_l0"] = stats["mean_degree_l0"]

        t0 = time.perf_counter()
        exact = exact_top10(X, Q, metric)
        res["exact_topk_s"] = time.perf_counter() - t0
        m = HNSW.load(folder)
        res["recall@10"] = {}
        for efS in EFS:
            idx, _ = m.predict(Q, pred_params=HNSW.PredParams(efS=efS, topk=10), ret_csr=False)
            res["recall@10"][str(efS)] = recall(idx, exact)
        del m

    if args.compare_reference:
        import oracle

        if not oracle.have_ref():
            res["reference"] = "not measured: oracle/_ref is absent"
        else:
            from oracle import ref

            t0 = time.perf_counter()
            r = ref.RefHNSW.train(X, M=M, efC=efC, metric=metric, threads=-1)
            rb = time.perf_counter() - t0
            rr = {}
            for efS in EFS:
                idx, _ = r.predict(Q, efS, 10, threads=-1)
                rr[str(efS)] = recall(idx, exact)
            res["reference"] = {"build_s": rb, "host_threads": os.cpu_count(), "recall@10": rr}
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, f"bench_hnsw_build_{args.workload}.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
