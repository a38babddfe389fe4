"""Sparse x sparse products on one H100: the PIFA product Z = Y^T X of the reference's examples/spmm benchmark through
c_sparse_matmul_csr_f32 with host buffers, against the reference library on the same inputs.

Workloads (seeds fixed here): X (N x D) and Y (N x L) at the N / D / L / nnz(X) / nnz(Y) of the reference's table for
eurlex-4k, amazoncat-13k and amazon-670k (--large adds wiki-500k and amazon-3m, which need far more host memory).  Each row of
X holds about nnz(X)/N distinct features drawn with p(f) ~ 1 / (f + 1)^1.1, each row of Y about nnz(Y)/N distinct labels
with p(l) ~ 1 / (l + 1)^1.2 (numpy default_rng(seed)); values uniform in [0.1, 1.1).  Y^T is converted to csr beforehand and
not timed; the call is sparse_matmul(Y^T, X, eliminate_zeros=False, sorted_indices=True) as in examples/spmm/run_exp.py.
Reported per workload: products (sum over Y^T entries of their X row lengths), nnz(Z), the C-ABI call (median of 5 after one
warm-up, host clock, result in host memory), kernel time (CUDA events, median of the same 5), products/s, compulsory bytes
(Y^T, X and Z read or written once) over kernel time against 3.35 TB/s, the reference library with all host cores (median
of 3) and with threads=1 (one run), the card name and power limit.
Parity gate (fails the run): indptr, indices and data up to indptr[-1], and the allocator nnz, byte-identical to oracle/_ref.
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

HBM_TBPS = 3.35
# name: (N, D, L, nnz(X), nnz(Y)) from the reference's examples/spmm/README.md
WORKLOADS = {
    "eurlex-4k": (15_449, 186_104, 3_956, 4_194_123, 82_265),
    "amazoncat-13k": (1_186_239, 203_882, 13_330, 84_415_397, 5_979_439),
    "amazon-670k": (490_449, 135_909, 670_091, 37_119_040, 2_674_356),
}
LARGE = {
    "wiki-500k": (1_779_881, 2_381_304, 501_070, 689_526_754, 8_446_236),
    "amazon-3m": (1_717_899, 337_067, 2_812_281, 84_600_285, 61_916_857),
}


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


def zipf_rows(rng, n, width, nnz, a):
    """n csr rows over [0, width) with about nnz entries in all, distinct per row, p(c) ~ 1 / (c + 1)^a."""
    p = 1.0 / (np.arange(width) + 1.0) ** a
    cdf = np.cumsum(p / p.sum())
    rows = np.sort(rng.integers(0, n, nnz))
    cols = np.minimum(np.searchsorted(cdf, rng.random(nnz)), width - 1)
    key = np.unique(rows.astype(np.int64) * width + cols)
    rows, cols = key // width, key % width
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.add.at(indptr, rows + 1, 1)
    data = (rng.random(key.size) + 0.1).astype(np.float32)
    return smat.csr_matrix((data, cols.astype(np.int32), np.cumsum(indptr)), shape=(n, width))


def make(name, shape):
    N, D, L, nx, ny = shape
    rng = np.random.default_rng(sum(map(ord, name)))
    X = zipf_rows(rng, N, D, nx, 1.1)
    Y = zipf_rows(rng, N, L, ny, 1.2)
    return smat.csr_matrix(Y.T, dtype=np.float32), X


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--large", action="store_true", help="also wiki-500k and amazon-3m (host memory: hundreds of GB)")
    ap.add_argument("--only", default=None, help="comma-separated workload names")
    ap.add_argument("--no-single-thread", action="store_true", help="skip the threads=1 reference run")
    args = ap.parse_args()

    from oracle import have_ref
    from pecos_b200 import core
    from tests import spmm_oracle as so

    lib = core.get_clib()
    lib.require_gpu()
    lib.set_device(0)
    if not have_ref():
        raise SystemExit("oracle/_ref is not built: the parity gate needs it")
    info_card = card()
    cores = os.cpu_count()
    todo = dict(WORKLOADS, **(LARGE if args.large else {}))
    if args.only:
        todo = {k: v for k, v in todo.items() if k in args.only.split(",")}
    failed = False
    for name, shape in todo.items():
        YT, X = make(name, shape)
        A, B = so.from_scipy(YT), so.from_scipy(X)
        got = so.call(lib.clib_float32, A, B, 0, 1)  # warm-up
        times, kms = [], []
        for _ in range(5):
            t0 = time.perf_counter()
            got = so.call(lib.clib_float32, A, B, 0, 1)
            times.append(time.perf_counter() - t0)
            kms.append(lib.clib_float32.pb200_spmm_last_kernel_ms())
        info = lib.sparse_matmul_last_info()
        ref_times = []
        for _ in range(3):
            t0 = time.perf_counter()
            want = so.reference(A, B, 0, 1, threads=cores)
            ref_times.append(time.perf_counter() - t0)
        t1 = None
        if not args.no_single_thread:
            t0 = time.perf_counter()
            so.reference(A, B, 0, 1, threads=1)
            t1 = time.perf_counter() - t0
        try:
            so.assert_same(got, want, name)
            parity = True
        except AssertionError as e:
            parity, failed = False, True
            print(str(e)[:500], file=sys.stderr)
        kernel_ms = float(np.median(kms))
        nnz_z = int(got["indptr"][-1])
        bytes_alg = 12 * (YT.nnz + X.nnz + nnz_z) + 8 * (2 * YT.shape[0] + X.shape[0] + 3)
        print(json.dumps({
            "workload": name, "shape": {"N": shape[0], "D": shape[1], "L": shape[2], "nnz_X": int(X.nnz),
                                        "nnz_Y": int(YT.nnz)},
            "products": info["products"], "nnz_Z": nnz_z, "tiers": {k: info[k] for k in (
                "count_warp_rows", "count_cta_rows", "fold_warp_rows", "fold_cta_rows")}, "tiles": info["tiles"],
            "call_s_median": float(np.median(times)), "kernel_ms_median": kernel_ms,
            "products_per_s": info["products"] / (kernel_ms / 1e3) if kernel_ms > 0 else None,
            "compulsory_bytes": bytes_alg, "hbm_share": bytes_alg / (kernel_ms / 1e3) / (HBM_TBPS * 1e12) if kernel_ms > 0 else None,
            "ref_all_cores_s_median": float(np.median(ref_times)), "ref_cores": cores, "ref_threads1_s": t1,
            "parity": parity, "card": info_card,
        }), flush=True)
    if failed:
        raise SystemExit("parity gate failed")


if __name__ == "__main__":
    main()
