"""GPU parity tests for the HNSW hot path: CUDA engine (through the C ABI / Python mirror) vs the CPU oracles.

Bar: bit-exact neighbour ids and ranks; distances bit-exact when the oracle ran the avx512f summation order the kernel
restates (the reference picks its SIMD clone at run time), else within 1e-5 relative.

Mirrors test/pecos/ann/test_hnsw.py: load -> predict identity incl. lazy_load (:20-56), recall vs brute force on the
prebuilt fixture index for efS in {50, 75, 100} (:58-124).
"""
import json
import os

import numpy as np
import pytest

from .util import save_hnsw_index

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hnsw_toy")


def _load(folder, **kw):
    from pecos_b200.hnsw import HNSW

    return HNSW.load(folder, **kw)


def _pp(efS, topk):
    from pecos_b200.hnsw import HNSW

    return HNSW.PredParams(efS=efS, topk=topk, threads=1)


@pytest.fixture(scope="module")
def golden(gpu_clib):
    E = np.load(os.path.join(GOLD, "expected.npz"))
    index = json.load(open(os.path.join(GOLD, "expected_index.json")))
    return E, index, np.load(os.path.join(GOLD, "X.tst.npy")), np.load(os.path.join(GOLD, "X.trn.npy"))


def test_golden_vectors_from_the_reference(golden):
    """Every recorded (model, efS, topk): ids, order and distance BITS (goldens were produced by the avx512f clone)."""
    E, index, Xt, _ = golden
    models = {}
    for it in index:
        m = models.get(it["model"]) or models.setdefault(it["model"], _load(os.path.join(GOLD, it["model"])))
        idx, dist = m.predict(Xt, pred_params=_pp(it["efS"], it["topk"]), ret_csr=False)
        assert np.array_equal(idx, E[it["key"] + "|idx"]), it["key"]
        assert np.array_equal(dist.view(np.uint32), E[it["key"] + "|dist"].view(np.uint32)), it["key"]


def test_load_predict_identity_lazy_and_searchers(golden):
    E, index, Xt, _ = golden
    a = _load(os.path.join(GOLD, "model_ip"))
    b = _load(os.path.join(GOLD, "model_ip"), lazy_load=True)
    s = a.searchers_create(2)
    ia, da = a.predict(Xt, pred_params=_pp(50, 10), searchers=s, ret_csr=False)
    ib, db = b.predict(Xt, pred_params=_pp(50, 10), ret_csr=False)
    assert np.array_equal(ia, ib) and np.array_equal(da, db)
    Y = a.predict(Xt, pred_params=_pp(50, 10), ret_csr=True)
    assert Y.shape == (Xt.shape[0], 90) and Y.nnz == Xt.shape[0] * 10
    with pytest.raises(ValueError):
        a.searchers_create(0)
    with pytest.raises(ValueError):
        a.predict(np.zeros((2, 5), dtype=np.float32))


def test_recall_against_brute_force(golden):
    E, index, Xt, Xtrn = golden
    m = _load(os.path.join(GOLD, "model_ip"))
    exact = np.argsort(1.0 - Xt @ Xtrn.T, axis=1, kind="stable")[:, :10]
    for efS in (50, 75, 100):
        idx, _ = m.predict(Xt, pred_params=_pp(efS, 10), ret_csr=False)
        recall = np.mean([len(set(idx[i]) & set(exact[i])) / 10.0 for i in range(Xt.shape[0])])
        assert recall == pytest.approx(1.0, abs=1e-2)


MID = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hnsw_mid")


def test_mid_size_golden_indices_from_the_reference(gpu_clib):
    """Reference-built indices with d in {768, 128, 70, 20} (tests/golden/make_golden_hnsw.py): 16-lane main loop, permuted
    layout, 4-wide remainder + scalar tail, real-sized TMA rows, six-fold exact ties, efS up to 600 -- ids, order and distance
    BITS as recorded from the reference library (avx512f clone).  Needs no oracle/_ref at test time."""
    E = np.load(os.path.join(MID, "expected.npz"))
    index = json.load(open(os.path.join(MID, "expected_index.json")))
    models = {}
    for it in index:
        folder = os.path.join(MID, it["model"])
        m = models.get(it["model"]) or models.setdefault(it["model"], _load(folder))
        Q = np.load(os.path.join(folder, "Q.npy"))
        idx, dist = m.predict(Q, pred_params=_pp(it["efS"], it["topk"]), ret_csr=False)
        assert np.array_equal(idx, E[it["key"] + "|idx"]), it["key"]
        assert np.array_equal(dist.view(np.uint32), E[it["key"] + "|dist"].view(np.uint32)), it["key"]


def test_mid_size_goldens_all_ring_depths(gpu_clib):
    """The same goldens with direct loads (0) and both bulk-copy ring depths (4, 8)."""
    E = np.load(os.path.join(MID, "expected.npz"))
    c = gpu_clib.clib_float32
    for name in ("ip_d768", "ip_d70", "l2_dup"):
        folder = os.path.join(MID, name)
        m = _load(folder)
        Q = np.load(os.path.join(folder, "Q.npy"))
        for stages in (0, 8, 4):
            assert c.pb200_hnsw_set_stages(m.model_ptr, stages) == stages
            idx, dist = m.predict(Q, pred_params=_pp(200, 10), ret_csr=False)
            assert np.array_equal(idx, E[f"{name}|200|10|idx"]), (name, stages)
            assert np.array_equal(dist.view(np.uint32), E[f"{name}|200|10|dist"].view(np.uint32)), (name, stages)


@pytest.mark.parametrize("N,d,M,metric", [(4000, 64, 8, "ip"), (3000, 70, 12, "l2"), (2500, 128, 16, "ip"),
                                          (1200, 3, 4, "l2"), (6000, 768, 16, "ip"), (2000, 100, 6, "l2")])
def test_random_indices_match_reference_library(tmp_path, gpu_clib, have_ref, N, d, M, metric):
    """Random indices (util.save_hnsw_index); the same saved index searched by the reference (where built), the restatement and us."""
    from oracle import restatement

    rng = np.random.default_rng(N + d)
    X = rng.standard_normal((N, d)).astype(np.float32)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    Q = rng.standard_normal((257, d)).astype(np.float32)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    folder = str(tmp_path / "idx")
    r = save_hnsw_index(folder, X, M, 60, metric, have_ref)
    m = _load(folder)
    o = restatement.OracleHNSW(folder, isa=0)  # avx512f order == what the kernel restates
    isa = restatement.host_isa()
    for efS, topk in [(10, 10), (64, 10), (200, 10), (5, 40), (600, 100)]:
        idx, dist = m.predict(Q, pred_params=_pp(efS, topk), ret_csr=False)
        oi, od = o.predict(Q, efS, topk)
        assert np.array_equal(idx, oi), f"ids vs restatement efS={efS} topk={topk}"
        assert np.array_equal(dist.view(np.uint32), od.view(np.uint32)), f"distance bits vs restatement efS={efS}"
        if r is None:
            continue
        ri, rd = r.predict(Q, efS, topk, threads=8)
        if isa == 0:
            assert np.array_equal(idx, ri) and np.array_equal(dist.view(np.uint32), rd.view(np.uint32)), "vs reference"
        else:  # the reference ran another SIMD clone: summation order differs in the last bits
            assert np.mean(idx == ri) > 0.99 and np.allclose(dist, rd, rtol=1e-5, atol=1e-6)


def test_duplicate_points_and_ties(tmp_path, gpu_clib, have_ref):
    """Many exactly equal distances: the restated libstdc++ heap algorithms decide which duplicates survive."""
    from oracle import restatement

    rng = np.random.default_rng(7)
    base = rng.standard_normal((300, 32)).astype(np.float32)
    base /= np.linalg.norm(base, axis=1, keepdims=True)
    X = np.concatenate([base] * 6, axis=0)  # every point six times
    Q = base[:64] + 0.0
    folder = str(tmp_path / "idx")
    r = save_hnsw_index(folder, X, 8, 50, "l2", have_ref, threads=1)
    m = _load(folder)
    for efS, topk in [(30, 12), (100, 20)]:
        idx, dist = m.predict(Q, pred_params=_pp(efS, topk), ret_csr=False)
        oi, od = restatement.OracleHNSW(folder, isa=0).predict(Q, efS, topk)
        assert np.array_equal(idx, oi) and np.array_equal(dist.view(np.uint32), od.view(np.uint32))
        if r is not None and restatement.host_isa() == 0:
            ri, rd = r.predict(Q, efS, topk, threads=1)
            assert np.array_equal(idx, ri) and np.array_equal(dist.view(np.uint32), rd.view(np.uint32))


def test_bulk_copy_ring_depths_give_identical_results(tmp_path, gpu_clib, have_ref):
    """0 = direct loads, 4 / 8 = base vectors staged through the per-warp TMA bulk-copy ring: same bits."""
    rng = np.random.default_rng(5)
    X = rng.standard_normal((5000, 200)).astype(np.float32)   # d = 200: permuted main part + 8-element tail
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    Q = rng.standard_normal((300, 200)).astype(np.float32)
    folder = str(tmp_path / "idx")
    save_hnsw_index(folder, X, 12, 60, "ip", have_ref)
    m = _load(folder)
    c = gpu_clib.clib_float32
    ref_out = None
    for stages in (0, 4, 8, 4):
        assert c.pb200_hnsw_set_stages(m.model_ptr, stages) == stages
        out = m.predict(Q, pred_params=_pp(100, 10), ret_csr=False)
        if ref_out is None:
            ref_out = out
        assert np.array_equal(out[0], ref_out[0]) and np.array_equal(out[1].view(np.uint32), ref_out[1].view(np.uint32))


def test_resident_batch_and_counters(golden, gpu_clib):
    from ctypes import POINTER, byref, c_float, c_uint32, c_uint64

    from oracle import restatement
    from pecos_b200.core import ScipyDrmF32

    E, index, Xt, _ = golden
    m = _load(os.path.join(GOLD, "model_l2"))
    c = gpu_clib.clib_float32
    px = ScipyDrmF32.init_from(np.ascontiguousarray(Xt))
    c.pb200_hnsw_resident_upload(m.model_ptr, byref(px))
    ms = c.pb200_hnsw_resident_predict(m.model_ptr, 50, 10)
    assert ms > 0
    idx = np.zeros((Xt.shape[0], 10), dtype=np.uint32)
    val = np.zeros((Xt.shape[0], 10), dtype=np.float32)
    c.pb200_hnsw_resident_fetch(m.model_ptr, idx.ctypes.data_as(POINTER(c_uint32)), val.ctypes.data_as(POINTER(c_float)))
    assert np.array_equal(idx, E["model_l2|50|10|idx"])
    cnt = (c_uint64 * 4)()
    c.pb200_hnsw_get_counters(m.model_ptr, cnt)
    oi, od, oc = restatement.OracleHNSW(os.path.join(GOLD, "model_l2"), isa=0).predict(Xt, 50, 10, return_counters=True)
    assert [int(x) for x in cnt] == [int(oc[:, 0].sum()), int(oc[:, 1].sum()), int(oc[:, 2].sum()), Xt.shape[0]]


def test_candidate_queue_overflow_is_retried_not_fatal(gpu_clib):
    """PB200_HNSW_VCAP=64 cannot hold the candidate queue of an efS = 600 search: the engine must re-run the batch with a larger
    queue (no abort) and return the recorded reference results."""
    import subprocess
    import sys

    code = ("import os, sys, numpy as np; sys.path.insert(0, %r); os.environ['PB200_HNSW_VCAP'] = '64'\n"
            "from pecos_b200.hnsw import HNSW; from pecos_b200 import core\n"
            "m = HNSW.load(%r); Q = np.load(%r); E = np.load(%r)\n"
            "idx, dist = m.predict(Q, pred_params=HNSW.PredParams(efS=600, topk=10, threads=1), ret_csr=False)\n"
            "assert np.array_equal(idx, E['ip_d70|600|10|idx']) and np.array_equal(dist.view(np.uint32), E['ip_d70|600|10|dist'].view(np.uint32))\n"
            "r = core.get_clib().clib_float32.pb200_hnsw_vcap_retries(m.model_ptr); assert r >= 1, r; print('retries', r)"
            % (os.path.dirname(os.path.dirname(os.path.abspath(__file__))), os.path.join(MID, "ip_d70"),
               os.path.join(MID, "ip_d70", "Q.npy"), os.path.join(MID, "expected.npz")))
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0 and "retries" in r.stdout, r.stderr[-1500:]


def test_resident_batch_survives_host_buffer_calls(golden, gpu_clib):
    """The resident batch and its results have their own device buffers: host-buffer searches in between, one larger and
    one smaller than the resident batch, change neither what resident_fetch returns nor the next resident_predict."""
    from ctypes import POINTER, byref, c_float, c_uint32

    from pecos_b200.core import ScipyDrmF32

    E, _, Xt, _ = golden
    m = _load(os.path.join(GOLD, "model_l2"))
    c = gpu_clib.clib_float32
    px = ScipyDrmF32.init_from(np.ascontiguousarray(Xt))
    c.pb200_hnsw_resident_upload(m.model_ptr, byref(px))

    def fetch():
        idx = np.zeros((Xt.shape[0], 10), dtype=np.uint32)
        val = np.zeros((Xt.shape[0], 10), dtype=np.float32)
        c.pb200_hnsw_resident_fetch(m.model_ptr, idx.ctypes.data_as(POINTER(c_uint32)), val.ctypes.data_as(POINTER(c_float)))
        return idx, val.view(np.uint32)

    c.pb200_hnsw_resident_predict(m.model_ptr, 50, 10)
    idx, val = fetch()
    assert np.array_equal(idx, E["model_l2|50|10|idx"])
    m.predict(np.ascontiguousarray(np.vstack([Xt, Xt, Xt])), pred_params=_pp(100, 20), ret_csr=False)
    m.predict(np.ascontiguousarray(Xt[:3]), pred_params=_pp(50, 5), ret_csr=False)
    for what in ("fetch", "resident_predict"):
        if what == "resident_predict":
            c.pb200_hnsw_resident_predict(m.model_ptr, 50, 10)
        i2, v2 = fetch()
        assert np.array_equal(i2, idx) and np.array_equal(v2, val), f"{what} after host-buffer calls"
