#!/usr/bin/env python
"""Generates tests/golden/hnsw_nonfinite/: REFERENCE-built HNSW indices whose stored rows then get NaN / overflowing values
written into the saved file (tests/hnsw_nonfinite_util.py), their queries, and the reference's search results.

  dense_ip_d70   N = 500, d = 70 (main chunk, 4-wide remainder, scalar tail), "scattered" rows incl. the order-dependent one
                                                                                          M = 12, efC = 40, metric ip
  dense_l2_d70   the same rows and edits, metric l2
  sparse_ip      N = 500 csr rows over 6,000 columns, sparse edits, a 5,000-entry query  M = 12, efC = 40, metric ip

Runs only where oracle/_ref/libpecos_float32.so is built.  Indices are trained single-threaded by the reference, saved, edited,
re-loaded and searched by the reference; ids and distance BITS are recorded (NaN payloads as the reference's x86 code left them).
"""
import json
import os
import shutil
import sys

import numpy as np
import scipy.sparse as smat

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

GRID = [(10, 10), (64, 10), (5, 40), (512, 10), (513, 10), (600, 100)]


def main():
    import oracle
    from oracle import ref, restatement
    from tests import hnsw_nonfinite_util as nf
    from tests.util import save_hnsw_index

    assert oracle.have_ref(), "build oracle/_ref first (make -C oracle)"
    assert restatement.host_isa() == 0, "record on a CPU where the reference runs its avx512f clone"
    out = os.path.join(HERE, "hnsw_nonfinite")
    shutil.rmtree(out, ignore_errors=True)
    os.makedirs(out)
    expected, index = {}, []
    cases = []
    for metric in ("ip", "l2"):
        rng = np.random.default_rng(500)
        X = nf.dense_rows(rng, 500, 70)
        Q, _ = nf.dense_queries(rng, 70, nq=8)
        cases.append((f"dense_{metric}_d70", X, Q, metric, lambda o, m=metric: nf.dense_edits(o, 70, m, "scattered")[0]))
    rng = np.random.default_rng(501)
    X = nf.sparse_rows(rng, 500)
    cases.append(("sparse_ip", X, nf.sparse_queries(rng, nq=8), "ip", nf.sparse_edits(X, 5)))
    for name, X, Q, metric, edits in cases:
        folder = os.path.join(out, name)
        save_hnsw_index(folder, X, 12, 40, metric, True, threads=1)
        nf.overwrite_values(folder, edits(restatement.OracleHNSW(folder)) if callable(edits) else edits)
        sparse = smat.issparse(X)
        if sparse:
            smat.save_npz(os.path.join(folder, "Q.npz"), Q)
        else:
            np.save(os.path.join(folder, "Q.npy"), Q)
        r = ref.RefHNSW.load(os.path.join(folder, "c_model"), metric, data_type="csr" if sparse else "drm")
        for efS, topk in GRID:
            idx, dist = r.predict(Q, efS, topk, threads=1)
            key = f"{name}|{efS}|{topk}"
            expected[key + "|idx"] = idx.astype(np.uint32)
            expected[key + "|dist"] = dist.astype(np.float32)
            index.append({"key": key, "model": name, "efS": efS, "topk": topk})
    np.savez_compressed(os.path.join(out, "expected.npz"), **expected)
    json.dump(index, open(os.path.join(out, "expected_index.json"), "w"), indent=1)
    json.dump({"grid": GRID, "distance_isa_clone": "avx512f",
               "note": "indices trained (threads=1) and saved by the unmodified reference library, then stored values "
                       "overwritten (tests/hnsw_nonfinite_util.py), re-loaded and searched by the reference"},
              open(os.path.join(out, "provenance.json"), "w"), indent=1)
    print("written", out)


if __name__ == "__main__":
    main()
