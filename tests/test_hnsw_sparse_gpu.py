"""GPU parity tests for SPARSE (csr) HNSW indices: CUDA engine through the C ABI / Python mirror vs the reference-recorded
goldens (tests/golden/hnsw_sparse), the C restatement and -- on freshly trained indices -- the reference library itself.

Bar: neighbour ids, order and distance BITS (the sparse intersection sums the matched products in ascending index order in
every SIMD clone of the reference, so there is no per-ISA tolerance here).

Mirrors test/pecos/ann/test_hnsw.py:86-124 (sparse fixture: load -> predict, recall vs brute force at efS in {50, 75, 100}).
"""
import importlib.util
import json
import os

import numpy as np
import pytest
import scipy.sparse as smat

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
SPARSE = os.path.join(HERE, "golden", "hnsw_sparse")


def _load(folder, **kw):
    from pecos_b200.hnsw import HNSW

    return HNSW.load(folder, **kw)


def _pp(efS, topk):
    from pecos_b200.hnsw import HNSW

    return HNSW.PredParams(efS=efS, topk=topk, threads=1)


def _rows():
    spec = importlib.util.spec_from_file_location("mgs", os.path.join(HERE, "golden", "make_golden_hnsw_sparse.py"))
    mgs = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mgs)
    return mgs.make_rows


def test_sparse_golden_indices_from_the_reference(gpu_clib):
    """Every recorded (index, efS, topk): the reference's own sparse fixture + three reference-built indices (ip, l2 = -2<x,y>,
    rows shorter than the 4-wide blocks, empty rows, a query row longer than every stored row)."""
    E = np.load(os.path.join(SPARSE, "expected.npz"))
    index = json.load(open(os.path.join(SPARSE, "expected_index.json")))
    models = {}
    for it in index:
        folder = os.path.join(SPARSE, it["model"])
        m = models.get(it["model"]) or models.setdefault(it["model"], _load(folder))
        assert m.data_type == "csr"
        Q = smat.load_npz(os.path.join(folder, "Q.npz"))
        idx, dist = m.predict(Q, pred_params=_pp(it["efS"], it["topk"]), ret_csr=False)
        assert np.array_equal(idx, E[it["key"] + "|idx"]), it["key"]
        assert np.array_equal(dist.view(np.uint32), E[it["key"] + "|dist"].view(np.uint32)), it["key"]


def test_sparse_fixture_recall_lazy_load_and_searchers(gpu_clib):
    from oracle import restatement

    fx = os.path.join(SPARSE, "fixture_ip")
    a, b = _load(fx), _load(fx, lazy_load=True)
    Q = smat.load_npz(os.path.join(fx, "Q.npz"))
    Xtrn = restatement.OracleHNSW(fx, isa=0).vectors()
    exact = np.argsort(1.0 - (Q @ Xtrn.T).toarray(), axis=1, kind="stable")[:, :10]
    s = a.searchers_create(2)
    for efS in (50, 75, 100):
        ia, da = a.predict(Q, pred_params=_pp(efS, 10), searchers=s, ret_csr=False)
        ib, db = b.predict(Q, pred_params=_pp(efS, 10), ret_csr=False)
        assert np.array_equal(ia, ib) and np.array_equal(da, db)
        recall = np.mean([len(set(ia[i]) & set(exact[i])) / 10.0 for i in range(Q.shape[0])])
        assert recall >= 0.99
    Y = a.predict(Q, pred_params=_pp(50, 10), ret_csr=True)
    assert Y.shape == (Q.shape[0], 90) and Y.nnz == Q.shape[0] * 10
    with pytest.raises(ValueError):
        a.predict(np.zeros((2, 2), dtype=np.float32))  # dense queries against a csr index
    with pytest.raises(ValueError):
        a.predict(smat.csr_matrix(np.ones((2, 5), dtype=np.float32)))  # wrong dimension
    # unsorted query indices are canonicalised by the Python layer (rows reversed here): same answer
    Qc = Q.copy()
    Qc.sort_indices()
    ind, dat = Qc.indices.copy(), Qc.data.copy()
    for i in range(Qc.shape[0]):
        s0, s1 = Qc.indptr[i], Qc.indptr[i + 1]
        ind[s0:s1], dat[s0:s1] = ind[s0:s1][::-1].copy(), dat[s0:s1][::-1].copy()
    Qu = smat.csr_matrix((dat, ind, Qc.indptr.copy()), shape=Q.shape, dtype=np.float32)
    assert not Qu.has_canonical_format
    iu, du = a.predict(Qu, pred_params=_pp(50, 10), ret_csr=False)
    ic, dc_ = a.predict(Qc, pred_params=_pp(50, 10), ret_csr=False)
    assert np.array_equal(iu, ic) and np.array_equal(du, dc_)


@pytest.mark.parametrize("N,D,nnz,M,metric", [(5000, 30000, 80, 12, "ip"), (3000, 2000, 25, 8, "l2"), (2000, 40, 4, 6, "ip"),
                                               (2500, 100000, 300, 16, "ip")])
def test_random_sparse_indices_match_reference_library(tmp_path, gpu_clib, have_ref, N, D, nnz, M, metric):
    """Indices built by the reference on this box; the same saved index searched by the reference, the restatement and us."""
    if not have_ref:
        pytest.skip("needs the reference library (oracle/_ref) to train sparse indices; reference-built sparse indices are "
                    "covered by test_sparse_golden_indices_from_the_reference")
    from oracle import ref, restatement

    make_rows = _rows()
    X = make_rows(N + D, N, D, nnz, 61)
    Q = make_rows(N + D + 1, 300, D, nnz, 17, long_row=(11, min(D, 5000)))  # one row beyond the shared-memory staging capacity
    r = ref.RefHNSW.train(X, M=M, efC=60, metric=metric, threads=8)
    folder = str(tmp_path / "idx")
    r.save(os.path.join(folder, "c_model"))
    json.dump({"model": "HNSW", "data_type": "csr", "metric_type": metric, "num_item": N, "feat_dim": D,
               "pred_kwargs": {"efS": 50, "topk": 10, "threads": 1}}, open(os.path.join(folder, "param.json"), "w"))
    m = _load(folder)
    o = restatement.OracleHNSW(folder, isa=0)
    for efS, topk in [(10, 10), (64, 10), (200, 10), (5, 40), (600, 100)]:
        idx, dist = m.predict(Q, pred_params=_pp(efS, topk), ret_csr=False)
        oi, od = o.predict(Q, efS, topk)
        assert np.array_equal(idx, oi), f"ids vs restatement efS={efS} topk={topk}"
        assert np.array_equal(dist.view(np.uint32), od.view(np.uint32)), f"distance bits vs restatement efS={efS}"
        ri, rd = r.predict(Q, efS, topk, threads=8)
        assert np.array_equal(idx, ri) and np.array_equal(dist.view(np.uint32), rd.view(np.uint32)), "vs reference library"


def test_sparse_resident_batch_counters_and_save(tmp_path, gpu_clib):
    from ctypes import POINTER, byref, c_float, c_uint32, c_uint64

    from oracle import restatement
    from pecos_b200.core import ScipyCsrF32

    folder = os.path.join(SPARSE, "ip_tfidf")
    E = np.load(os.path.join(SPARSE, "expected.npz"))
    m = _load(folder)
    Q = smat.load_npz(os.path.join(folder, "Q.npz"))
    Q.sort_indices()
    c = gpu_clib.clib_float32
    px = ScipyCsrF32.init_from(Q)
    c.pb200_hnsw_resident_upload_csr(m.model_ptr, byref(px))
    ms = c.pb200_hnsw_resident_predict(m.model_ptr, 200, 10)
    assert ms > 0
    idx = np.zeros((Q.shape[0], 10), dtype=np.uint32)
    val = np.zeros((Q.shape[0], 10), dtype=np.float32)
    c.pb200_hnsw_resident_fetch(m.model_ptr, idx.ctypes.data_as(POINTER(c_uint32)), val.ctypes.data_as(POINTER(c_float)))
    assert np.array_equal(idx, E["ip_tfidf|200|10|idx"])
    assert np.array_equal(val.view(np.uint32), E["ip_tfidf|200|10|dist"].view(np.uint32))
    cnt = (c_uint64 * 4)()
    c.pb200_hnsw_get_counters(m.model_ptr, cnt)
    o = restatement.OracleHNSW(folder, isa=0)
    oi, od, oc = o.predict(Q, 200, 10, return_counters=True)
    assert [int(x) for x in cnt] == [int(oc[:, 0].sum()), int(oc[:, 1].sum()), int(oc[:, 2].sum()), Q.shape[0]]
    assert c.pb200_hnsw_sparse_entries(m.model_ptr) > 0
    # save = the files the index was loaded from; the copy loads and answers identically
    out = str(tmp_path / "copy")
    os.makedirs(out)
    m.fn_dict["save"](m.model_ptr, os.path.join(out, "c_model").encode())
    json.dump(json.load(open(os.path.join(folder, "param.json"))), open(os.path.join(out, "param.json"), "w"))
    m2 = _load(out)
    i2, d2 = m2.predict(Q, pred_params=_pp(200, 10), ret_csr=False)
    assert np.array_equal(i2, idx) and np.array_equal(d2, val)


def test_sparse_resident_batch_survives_host_buffer_calls(gpu_clib):
    """As for dense indices: host-buffer searches between the resident calls, one larger (more rows and longer rows, so the
    query staging grows) and one smaller, change neither what resident_fetch returns nor the next resident_predict."""
    from ctypes import POINTER, byref, c_float, c_uint32

    from pecos_b200.core import ScipyCsrF32

    folder = os.path.join(SPARSE, "ip_tfidf")
    E = np.load(os.path.join(SPARSE, "expected.npz"))
    m = _load(folder)
    Q = smat.load_npz(os.path.join(folder, "Q.npz")).tocsr()
    Q.sort_indices()
    c = gpu_clib.clib_float32
    px = ScipyCsrF32.init_from(Q)
    c.pb200_hnsw_resident_upload_csr(m.model_ptr, byref(px))

    def fetch():
        idx = np.zeros((Q.shape[0], 10), dtype=np.uint32)
        val = np.zeros((Q.shape[0], 10), dtype=np.float32)
        c.pb200_hnsw_resident_fetch(m.model_ptr, idx.ctypes.data_as(POINTER(c_uint32)), val.ctypes.data_as(POINTER(c_float)))
        return idx, val.view(np.uint32)

    c.pb200_hnsw_resident_predict(m.model_ptr, 200, 10)
    idx, val = fetch()
    assert np.array_equal(idx, E["ip_tfidf|200|10|idx"])
    # more rows, and longer ones: each row of `big` is the sum of two rows of Q
    both = (Q + Q[np.random.default_rng(7).permutation(Q.shape[0])]).tocsr()
    big = smat.vstack([both, both, both]).tocsr().astype(np.float32)
    big.sort_indices()
    assert big.shape[0] > Q.shape[0] and np.diff(big.indptr).max() > np.diff(Q.indptr).max()
    m.predict(big, pred_params=_pp(100, 20), ret_csr=False)
    m.predict(Q[:3], pred_params=_pp(50, 5), ret_csr=False)
    for what in ("fetch", "resident_predict"):
        if what == "resident_predict":
            c.pb200_hnsw_resident_predict(m.model_ptr, 200, 10)
        i2, v2 = fetch()
        assert np.array_equal(i2, idx) and np.array_equal(v2, val), f"{what} after host-buffer calls"
