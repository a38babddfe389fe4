"""PairwiseANN on one H100: pairs/s through the C ABI with host buffers, kernel time by CUDA events, algorithmic bytes against
3.35 TB/s, the replay-path share, and the reference library on the same inputs with all host cores.

Workloads (seeds fixed here):
  dense:  X = 1,000,000 x 768 standard-normal rows, L2-normalised (numpy default_rng(1)); queries default_rng(2), same law.
  sparse: X = bench.make_sparse_rows(30, 1,000,000, 47,236, 76) (the hnsw-rcv1 row shape), queries make_sparse_rows(31, ...).
  Y (both): 3 distinct labels per input drawn from p(l) ~ 1 / (l + 1)^0.9 over 200,000 labels (default_rng(3)), value 1;
  column lengths run from 1 to tens of thousands.  Label keys of the batch: the columns of uniformly drawn nonzeros of Y
  (i.e. by label frequency, default_rng(4)).  only_topk = 10, is_same_input = False.
Algorithmic bytes per pair: dense 16 + n (8 + 4d) + 4d (its query) + 16 topk; sparse 16 + n (8 + 16) + 8 (entries of the n rows)
+ 8 nnz(query) + 16 topk.
Parity gate (fails the run): I / M / D / V bit-equal to oracle/_ref on the first --gate pairs.
Prints one JSON line per workload.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse as smat

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from bench import make_sparse_rows  # noqa: E402

HBM_TBPS = 3.35


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


def make_y(N, L=200_000, per_row=3, a=0.9, seed=3):
    rng = np.random.default_rng(seed)
    p = 1.0 / (np.arange(L) + 1.0) ** a
    cdf = np.cumsum(p / p.sum())
    cols = np.searchsorted(cdf, rng.random((N, per_row * 2)))
    cols.sort(axis=1)
    keep = np.ones(cols.shape, bool)
    keep[:, 1:] = cols[:, 1:] != cols[:, :-1]
    rows = np.repeat(np.arange(N), cols.shape[1])[keep.ravel()]
    cols = cols.ravel()[keep.ravel()]
    first = np.zeros(rows.size, bool)  # keep the first per_row distinct labels of each row
    _, start = np.unique(rows, return_index=True)
    rank = np.arange(rows.size) - np.repeat(start, np.diff(np.append(start, rows.size)))
    first = rank < per_row
    Y = smat.csc_matrix((np.ones(first.sum(), np.float32), (rows[first], cols[first])), shape=(N, L))
    return Y


def workload(kind, N, d):
    if kind == "dense":
        X = np.random.default_rng(1).standard_normal((N, d), dtype=np.float32)
        X /= np.linalg.norm(X, axis=1, keepdims=True)
        return X
    return make_sparse_rows(30, N, d, 76)


def queries(kind, B, d):
    if kind == "dense":
        Q = np.random.default_rng(2).standard_normal((B, d), dtype=np.float32)
        Q /= np.linalg.norm(Q, axis=1, keepdims=True)
        return Q
    return make_sparse_rows(31, B, d, 76)


def run(kind, args):
    from oracle.pairwise import RefPairwise
    from pecos_b200.core import get_clib
    from pecos_b200.pairwise import PairwiseANN

    N, d = args.n, (768 if kind == "dense" else 47_236)
    X = workload(kind, N, d)
    Y = make_y(N)
    lens = np.diff(Y.indptr)
    nzcols = np.repeat(np.arange(Y.shape[1]), lens)
    keys = nzcols[np.random.default_rng(4).integers(0, nzcols.size, size=args.batch)].astype(np.uint32)
    Q = queries(kind, args.batch, d)
    n = lens[keys].astype(np.float64)
    topk = 10
    if kind == "dense":
        algo = float((16 + n * (8 + 4 * d) + 4 * d + 16 * topk).sum())
    else:
        row_nnz = np.diff(X.indptr)
        csum = np.concatenate([[0.0], np.cumsum(row_nnz[Y.indices].astype(np.float64))])
        ent = csum[Y.indptr[keys + 1]] - csum[Y.indptr[keys]]  # stored entries of each pair's column rows
        algo = float((16 + n * 24 + 8 * ent + 8 * np.diff(Q.indptr) + 16 * topk).sum())
    clib = get_clib()
    clib.set_device(0)
    model = PairwiseANN.train(X, Y)
    s = model.searchers_create(PairwiseANN.PredParams(batch_size=args.batch, only_topk=topk))
    model.predict(Q, keys, s)  # warm-up: uploads the model, loads the kernels
    walls, kms = [], []
    for _ in range(args.steps):
        t0 = time.perf_counter()
        I, M, D, V = [a.copy() for a in model.predict(Q, keys, s)]
        walls.append(time.perf_counter() - t0)
        kms.append(clib.clib_float32.pb200_pairwise_ann_kernel_ms(s.ctypes()))
    cnt = s.counters()
    # parity gate + reference timing on the first args.gate pairs, all host cores
    g = args.gate
    ref = RefPairwise.train(X, Y)
    threads = os.cpu_count()
    Qg = Q[:g]
    t0 = time.perf_counter()
    want = ref.predict(Qg, keys[:g], topk, False, threads=threads)
    ref_s = time.perf_counter() - t0
    s_g = model.searchers_create(PairwiseANN.PredParams(batch_size=g, only_topk=topk))
    got = model.predict(Qg, keys[:g], s_g)
    ok = all(np.array_equal(np.asarray(a).view(np.uint32), np.asarray(b).view(np.uint32)) for a, b in zip(got, want))
    wall = float(np.median(walls))
    kernel_ms = float(np.median(kms))
    out = {
        "workload": f"pairwise-{kind}", "N": N, "d": d, "labels": int(Y.shape[1]), "batch": args.batch, "topk": topk,
        "column_len_min_nonzero": int(lens[lens > 0].min()), "column_len_max": int(lens.max()),
        "mean_n_per_pair": float(n.mean()), "distances": cnt["distances"], "replay_pairs": cnt["replays"],
        "replay_share": cnt["replays"] / max(cnt["pairs"], 1), "sparse_entries": cnt["sparse_entries"],
        "pairs_per_s_c_abi": args.batch / wall, "wall_s_median": wall, "kernel_ms_median": kernel_ms,
        "algorithmic_bytes": algo, "kernel_tb_per_s": algo / (kernel_ms * 1e-3) / 1e12,
        "kernel_share_of_3.35TBps": algo / (kernel_ms * 1e-3) / 1e12 / HBM_TBPS,
        "reference_pairs": g, "reference_threads": threads, "reference_pairs_per_s": g / ref_s,
        "parity_gate_pairs": g, "parity_ok": ok, "card": card(),
    }
    print(json.dumps(out), flush=True)
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", choices=("dense", "sparse", "both"), default="both")
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--batch", type=int, default=20_000)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--gate", type=int, default=2000)
    args = ap.parse_args()
    ok = True
    for kind in (("dense", "sparse") if args.workload == "both" else (args.workload,)):
        ok = run(kind, args) and ok
    if not ok:
        print("parity gate FAILED: outputs differ from oracle/_ref", file=sys.stderr)
        sys.exit(1)


if __name__ == "__main__":
    main()
