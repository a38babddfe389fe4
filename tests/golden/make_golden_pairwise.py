"""Records tests/golden/pairwise_ann/ from the reference library (oracle/_ref/libpecos_float32.so).

Each case folder holds a reference-trained, reference-saved model (param.json as the reference's Python writes it, c_model/
written by c_pairwise_ann_save_*) and its queries; expected.npz holds the reference's I / M / D / V bits for every case,
only_topk in {0, 1, 10, longest column + 5} and is_same_input in {False, True} (keys "<case>|<topk>|<same>|<I,M,D,V>", label
keys under "<case>|keys").  Run from the repository root:  python tests/golden/make_golden_pairwise.py
"""
import json
import os
import sys

import numpy as np
import scipy.sparse as smat

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.pairwise import RefPairwise  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "pairwise_ann")


def zipf_csc(rng, N, L, per_row=3, a=1.3):
    """Y with a few labels per input drawn from a Zipf-like law over L labels; entries stored in a shuffled order."""
    rows, cols = [], []
    p = 1.0 / np.arange(1, L + 1) ** a
    p /= p.sum()
    for r in range(N):
        for c in rng.choice(L, size=per_row, replace=False, p=p):
            rows.append(r)
            cols.append(c)
    Y = smat.csc_matrix((np.round(rng.random(len(rows)) * 8 + 1).astype(np.float32) / 4, (rows, cols)), shape=(N, L))
    return Y


def raw_csc(cols, N, rng):
    """csc from explicit per-column row lists, stored exactly as listed (unsorted, duplicates kept)."""
    indptr = np.cumsum([0] + [len(c) for c in cols]).astype(np.int64)
    idx = np.array([r for c in cols for r in c], dtype=np.int32)
    val = (np.round(rng.random(idx.size) * 4 + 1) / 2).astype(np.float32)
    return smat.csc_matrix((val, idx, indptr), shape=(N, len(cols)))


def cases(rng):
    out = {}
    # dense d = 70: 16-lane main loop, 4-wide remainder and scalar tail of the distance
    N, L = 400, 30
    out["dense_d70"] = (rng.standard_normal((N, 70)).astype(np.float32), zipf_csc(rng, N, L), rng.standard_normal((48, 70)).astype(np.float32))
    # dense d = 768: 16-lane main loop only
    N, L = 150, 8
    out["dense_d768"] = (rng.standard_normal((N, 768)).astype(np.float32), zipf_csc(rng, N, L), rng.standard_normal((16, 768)).astype(np.float32))
    # sparse tf-idf-like rows
    N, L, d = 400, 30, 500
    X = smat.random(N, d, density=0.03, format="csr", dtype=np.float32, random_state=rng.integers(1 << 30))
    Q = smat.random(48, d, density=0.03, format="csr", dtype=np.float32, random_state=rng.integers(1 << 30))
    out["sparse"] = (X, zipf_csc(rng, N, L), Q)
    # dense ties: few-level values, duplicated rows, a row listed twice in a column, unsorted row indices, empty columns
    N, d = 60, 20
    X = rng.integers(-1, 2, size=(N, d)).astype(np.float32)
    X[30:40] = X[0:10]
    cols = [list(rng.permutation(N)[:k]) for k in (25, 40, 0, 7, 60, 1, 0, 33)]
    cols[1] = cols[1] + cols[1][:5]
    out["ties_dense"] = (X, raw_csc(cols, N, rng), rng.integers(-1, 2, size=(24, d)).astype(np.float32))
    # sparse ties: rows disjoint from the query (distance exactly 1.0) at the top-k boundary, duplicates, empty columns
    N, d = 80, 40
    dense = rng.integers(0, 3, size=(N, d)) * (rng.random((N, d)) < 0.08)
    dense[40:50] = dense[0:10]
    X = smat.csr_matrix(dense.astype(np.float32))
    cols = [list(rng.permutation(N)[:k]) for k in (30, 80, 0, 12, 55, 2)]
    cols[4] = cols[4] + cols[4][::3]
    Qd = rng.integers(0, 3, size=(24, d)) * (rng.random((24, d)) < 0.08)
    out["ties_sparse"] = (X, raw_csc(cols, N, rng), smat.csr_matrix(Qd.astype(np.float32)))
    # the reference's own test_predict_with_same_input (test/pecos/ann/test_pairwise_ann.py)
    X = np.array([[1, 0], [2, 0], [3, 0], [4, 0], [5, 0]], dtype=np.float32)
    Y = smat.csr_matrix(np.array([[1.1, 0, 0, 0], [2.1, 2.2, 0, 0], [0, 3.2, 3.3, 0], [0, 0, 4.3, 4.4], [0, 0, 0, 5.4]],
                                 dtype=np.float32)).tocsc()
    out["same_input"] = (X, Y, X[:4].copy())
    return out


def param_json(data_type, N, L, d):
    return {"__meta__": {"class_fullname": "pecos.ann.pairwise.model###PairwiseANN"}, "model": "PairwiseANN", "data_type": data_type,
            "metric_type": "ip", "num_input_keys": N, "num_label_keys": L, "feat_dim": d,
            "pred_kwargs": {"__meta__": {"class_fullname": "pecos.ann.pairwise.model###PairwiseANN.PredParams"}, "batch_size": 1024,
                            "only_topk": 10}}


def main():
    rng = np.random.default_rng(20261017)
    expected = {}
    for name, (X, Y, Q) in cases(rng).items():
        folder = os.path.join(OUT, name)
        os.makedirs(folder, exist_ok=True)
        data_type = "csr" if isinstance(X, smat.csr_matrix) else "drm"
        ref = RefPairwise.train(X, Y)
        ref.save(os.path.join(folder, "c_model"))
        with open(os.path.join(folder, "param.json"), "w") as f:
            f.write(json.dumps(param_json(data_type, X.shape[0], Y.shape[1], X.shape[1]), indent=True))
        if data_type == "csr":
            smat.save_npz(os.path.join(folder, "Q.npz"), Q, compressed=False)
        else:
            np.save(os.path.join(folder, "Q.npy"), Q)
        L = Y.shape[1]
        keys = np.concatenate([np.arange(L), rng.integers(0, L, size=Q.shape[0] - L)]) if Q.shape[0] > L else np.arange(Q.shape[0]) % L
        keys = keys.astype(np.uint32)
        expected[f"{name}|keys"] = keys
        longest = int(np.diff(Y.indptr).max())
        for topk in (0, 1, 10, longest + 5):
            for same in (False, True):
                for tag, a in zip("IMDV", ref.predict(Q, keys, topk, same)):
                    expected[f"{name}|{topk}|{int(same)}|{tag}"] = a.view(np.uint32) if a.dtype == np.float32 else a
    np.savez_compressed(os.path.join(OUT, "expected.npz"), **expected)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
