"""CPU tests of the SPARSE (csr) HNSW builder's host logic and file format (pecos_b200/hnsw_build.py with a scipy sparse input and
device="cpu" on tiny inputs; the GPU kernels are tests/test_hnsw_build_sparse_gpu.py).  The written index must parse, store the
canonicalised rows, respect the reference's structural invariants with neighbours ordered by the reference's sparse distance,
load in the REFERENCE library (oracle/_ref) with bit-identical searches, and recall at the level of a reference-trained index."""
import importlib.util
import json
import os
from ctypes import POINTER, c_float, c_uint32

import numpy as np
import pytest
import scipy.sparse as smat

HERE = os.path.dirname(os.path.abspath(__file__))


def make_rows(*a, **kw):
    spec = importlib.util.spec_from_file_location("mgs", os.path.join(HERE, "golden", "make_golden_hnsw_sparse.py"))
    mgs = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mgs)
    return mgs.make_rows(*a, **kw)


def with_duplicates(X, seed):
    """The same matrix written non-canonically: every 5th row gets a duplicate of its first entry (value 0.25) and every row's
    entries are stored in reverse order."""
    rng = np.random.default_rng(seed)
    indptr, idx, val = [0], [], []
    for i in range(X.shape[0]):
        c = X.indices[X.indptr[i]:X.indptr[i + 1]].tolist()
        v = X.data[X.indptr[i]:X.indptr[i + 1]].tolist()
        if c and i % 5 == 0:
            c.append(c[0])
            v.append(0.25)
        order = np.argsort(rng.random(len(c)))[::-1] if len(c) else []
        idx += [c[k] for k in order]
        val += [v[k] for k in order]
        indptr.append(len(idx))
    return smat.csr_matrix((np.array(val, dtype=np.float32), np.array(idx, dtype=np.int32), np.array(indptr)), shape=X.shape)


def sparse_distance(X, i, Y, j, metric):
    """The restatement's hno_sparse_distance (the reference's FeatVecSparse{IP,L2}Simd::distance) of X[i] and Y[j]."""
    from oracle import restatement

    L = restatement._hnsw_lib()
    xi, xv = X.indices[X.indptr[i]:X.indptr[i + 1]].astype(np.uint32), X.data[X.indptr[i]:X.indptr[i + 1]].astype(np.float32)
    yi, yv = Y.indices[Y.indptr[j]:Y.indptr[j + 1]].astype(np.uint32), Y.data[Y.indptr[j]:Y.indptr[j + 1]].astype(np.float32)
    return np.float32(L.hno_sparse_distance(xi.size, xv.ctypes.data_as(POINTER(c_float)), xi.ctypes.data_as(POINTER(c_uint32)),
                                            yi.size, yv.ctypes.data_as(POINTER(c_float)), yi.ctypes.data_as(POINTER(c_uint32)),
                                            {"ip": 0, "l2": 1}[metric], 0))


def exact_topk(Q, X, metric, k=10):
    dot = (Q @ X.T).toarray().astype(np.float64)
    return np.argsort((1.0 - dot) if metric == "ip" else -2.0 * dot, axis=1, kind="stable")[:, :k]


def recall(idx, exact):
    return float(np.mean([len(set(idx[i].tolist()) & set(exact[i].tolist())) / exact.shape[1] for i in range(idx.shape[0])]))


# floor: the recall@10 (efS = 80) of the reference-trained index on the same rows and queries, minus 0.02 (measured: 0.885, 0.847,
# 0.924; exact ties among rows sharing no feature with the query keep these low for both builders)
@pytest.mark.parametrize("N,D,nnz,M,efC,metric,floor", [(1500, 3000, 20, 5, 40, "ip", 0.86), (1000, 500, 12, 4, 30, "l2", 0.82),
                                                         (60, 40, 4, 3, 10, "ip", 0.90)])
def test_sparse_index_format_graph_and_recall(tmp_path, built, have_ref, N, D, nnz, M, efC, metric, floor):
    from oracle import restatement
    from pecos_b200.hnsw_build import build_hnsw_index

    base = make_rows(N + D, N, D, nnz, 37)                      # every 37th row is empty
    X = with_duplicates(base, N)
    assert not X.has_canonical_format
    Xc = X.copy()
    Xc.sum_duplicates()
    Xc.sort_indices()
    Q = make_rows(N + D + 1, 80, D, nnz, 0, long_row=(3, min(D, 8 * nnz)))
    folder = str(tmp_path / "idx")
    stats = build_hnsw_index(X, folder, M=M, efC=efC, metric=metric, seed=7, device="cpu", q_tile=256, c_tile=600, h_tile=64)
    assert stats["num_node"] == N and stats["feat_dim"] == D
    if N >= 1000:
        assert stats["max_level"] >= 2
    cfg = json.load(open(os.path.join(folder, "c_model", "config.json")))
    kind = "IP" if metric == "ip" else "L2"
    assert cfg["hnsw_t"] == f"pecos::ann::HNSW<float, pecos::ann::FeatVecSparse{kind}Simd<uint32_t, float>>"
    assert cfg["version"] == "v2.0" and cfg["train_params"]["maxM0"] == 2 * M and cfg["train_params"]["maxM"] == M
    param = json.load(open(os.path.join(folder, "param.json")))
    assert param["data_type"] == "csr" and param["metric_type"] == metric
    assert param["num_item"] == N and param["feat_dim"] == D

    o = restatement.OracleHNSW(folder, isa=0)
    assert o.sparse and o.l0_node_mem == 0 and o.feat_dim == D and o.num_node == N
    V = o.vectors()
    assert np.array_equal(V.indptr, Xc.indptr) and np.array_equal(V.indices, Xc.indices)
    assert np.array_equal(V.data.view(np.uint32), Xc.data.view(np.uint32))
    # level 0: degree within capacity, no self loops, no duplicates, ascending by the reference's sparse distance
    for u in range(N):
        b = int(o.mem_start[u])
        deg = int(o.l0[b:b + 4].view(np.uint32)[0])
        assert deg <= 2 * M
        nb = o.l0[b + 4:b + 4 + 4 * deg].view(np.uint32)
        assert u not in nb and len(set(nb.tolist())) == deg and np.all(nb < N)
        dist = np.array([sparse_distance(Xc, u, Xc, int(v), metric) for v in nb], dtype=np.float32)
        assert np.all(dist[1:] >= dist[:-1]), u
    # upper levels
    l1 = o.l1.view(np.uint32)
    for lvl in range(1, o.max_level + 1):
        for u in range(0, N, 7):
            s = u * o.l1_node_mem + (lvl - 1) * o.l1_level_mem
            if s >= l1.size:
                continue
            deg = int(l1[s])
            nb = l1[s + 1:s + 1 + deg]
            assert deg <= M and u not in nb and len(set(nb.tolist())) == deg

    oi, od = o.predict(Q, 80, 10)
    exact = exact_topk(Q, Xc, metric)
    r = recall(oi, exact)
    assert r >= floor, r
    if have_ref:
        from oracle import ref

        rl = ref.RefHNSW.load(os.path.join(folder, "c_model"), metric, data_type="csr")  # the REFERENCE loads our file
        ri, rd = rl.predict(Q, 80, 10, threads=1)
        assert np.array_equal(ri, oi) and np.array_equal(rd.view(np.uint32), od.view(np.uint32))
        trained = ref.RefHNSW.train(Xc, M=M, efC=efC, metric=metric, threads=1)
        ti, _ = trained.predict(Q, 80, 10, threads=1)
        assert r >= recall(ti, exact) - 0.02, (r, recall(ti, exact))


def test_sparse_input_errors(tmp_path):
    from pecos_b200.hnsw_build import build_hnsw_index

    with pytest.raises(ValueError):
        build_hnsw_index(smat.csr_matrix((0, 10), dtype=np.float32), str(tmp_path / "a"), device="cpu")
    X = make_rows(5, 20, 30, 4, 0)
    with pytest.raises(ValueError):
        build_hnsw_index(X, str(tmp_path / "b"), metric="cos", device="cpu")
    with pytest.raises(ValueError):
        build_hnsw_index(X, str(tmp_path / "c"), efC=513, device="cpu")
