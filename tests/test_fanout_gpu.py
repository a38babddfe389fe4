"""In-library multi-GPU query fan-out (SURVEY 8e): PB200_DEVICES lists the devices that get a replica of the model at load
time; one predict call then splits its rows over the replicas (one host thread + stream per device) and concatenates the
results in row order.  Here a world of 2-3 is emulated on ONE GPU by listing device 0 several times; the result must be
bit-identical to the single-engine call (rows are independent: reference analogue inference.hpp:969-1005)."""
import os

import numpy as np
import pytest

from pecos_b200 import synth

from .util import assert_csr_parity, csr_with_empty_rows, random_tree

pytestmark = pytest.mark.gpu

MID = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hnsw_mid")


@pytest.fixture()
def devices_env():
    old = os.environ.get("PB200_DEVICES")
    yield
    if old is None:
        os.environ.pop("PB200_DEVICES", None)
    else:
        os.environ["PB200_DEVICES"] = old


def test_xlinear_fanout_equals_single_engine(tmp_path, gpu_clib, devices_env):
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    layers = random_tree(211, [6, 40, 700], 600, 30, bias=1.0, permute=True, prune=0.1)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=8)
    X = synth.make_queries(212, 2100, 600, 50)
    X = csr_with_empty_rows(X, [0, 1, 2, 1000, 2099])  # ragged rows incl. empty ones at both ends
    c = gpu_clib.clib_float32
    os.environ.pop("PB200_DEVICES", None)
    single = XLinearModel.load(folder, is_predict_only=True)
    assert c.pb200_xlinear_replicas(single.model.model_chain) == 1
    want = single.predict(X, beam_size=7, only_topk=6)
    want_d = single.predict(X[:900].toarray(), beam_size=7, only_topk=6)
    for devs, n in (("0,0", 2), ("0,0,0", 3)):
        os.environ["PB200_DEVICES"] = devs
        m = XLinearModel.load(folder, is_predict_only=True)
        assert c.pb200_xlinear_replicas(m.model.model_chain) == n
        assert_csr_parity(m.predict(X, beam_size=7, only_topk=6), want, rtol=0.0, what=f"csr fan-out {devs}")
        assert_csr_parity(m.predict(X[:900].toarray(), beam_size=7, only_topk=6), want_d, rtol=0.0, what=f"dense fan-out {devs}")
        # small batches are served by one engine; must still be right
        assert_csr_parity(m.predict(X[:50], beam_size=7, only_topk=6), want[:50], rtol=0.0, what=f"small batch {devs}")
        # rows shorter than k (ragged result rows) cross the device boundaries
        assert_csr_parity(m.predict(X, beam_size=2, only_topk=500), single.predict(X, beam_size=2, only_topk=500), rtol=0.0,
                          what=f"ragged result rows {devs}")


def test_xlinear_fanout_through_both_csr_schedules(tmp_path, gpu_clib, devices_env, monkeypatch):
    """10,000 CSR rows over two replicas: each replica's row block holds >= 4096 rows, and the second one starts at
    row_ptr[0] != 0.  At the default workspace each block takes the whole-batch upload schedule; at PB200_WORKSPACE_MB=64
    (about 1,000 queries per tile at beam 64 over 16,384 labels) the two-set schedule.  Both equal one engine bit for bit."""
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path / "m")
    layers = random_tree(231, [64, 16384], 300, 20, bias=1.0)
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=10)
    X = synth.make_queries(232, 10000, 300, 30)
    c = gpu_clib.clib_float32
    monkeypatch.delenv("PB200_WORKSPACE_MB", raising=False)
    os.environ.pop("PB200_DEVICES", None)
    want = XLinearModel.load(folder, is_predict_only=True).predict(X, beam_size=64, only_topk=10)
    os.environ["PB200_DEVICES"] = "0,0"
    m = XLinearModel.load(folder, is_predict_only=True)
    h = m.model.model_chain
    assert c.pb200_xlinear_replicas(h) == 2
    launches = []
    for mb in (None, "64"):
        if mb:
            monkeypatch.setenv("PB200_WORKSPACE_MB", mb)
        l0 = c.pb200_xlinear_launches(h)
        got = m.predict(X, beam_size=64, only_topk=10)
        launches.append(c.pb200_xlinear_launches(h) - l0)
        assert assert_csr_parity(got, want, rtol=0.0, what=f"fan-out 0,0, workspace {mb or 'default'} MiB") == 1.0
    assert launches[1] > launches[0], f"launches {launches}: the 64 MiB workspace did not cut the blocks into tiles"


def test_hnsw_fanout_equals_single_engine(gpu_clib, devices_env):
    from pecos_b200.hnsw import HNSW

    folder = os.path.join(MID, "l2_d128")
    Q = np.load(os.path.join(folder, "Q.npy"))
    rng = np.random.default_rng(5)
    Qbig = np.ascontiguousarray(np.concatenate([Q] * 12 + [rng.standard_normal((33, Q.shape[1])).astype(np.float32)]))
    os.environ.pop("PB200_DEVICES", None)
    single = HNSW.load(folder)
    want = single.predict(Qbig, pred_params=HNSW.PredParams(efS=100, topk=10, threads=1), ret_csr=False)
    os.environ["PB200_DEVICES"] = "0,0,0"
    m = HNSW.load(folder)
    assert gpu_clib.clib_float32.pb200_hnsw_replicas(m.model_ptr) == 3
    got = m.predict(Qbig, pred_params=HNSW.PredParams(efS=100, topk=10, threads=1), ret_csr=False)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))


def test_sparse_hnsw_fanout_equals_single_engine(gpu_clib, devices_env):
    """csr queries: every replica gets its rows of the caller's csr arrays (row offsets rebased per slice)."""
    import scipy.sparse as smat

    from pecos_b200.hnsw import HNSW

    folder = os.path.join(os.path.dirname(MID), "hnsw_sparse", "ip_tfidf")
    Q = smat.load_npz(os.path.join(folder, "Q.npz"))
    Qbig = smat.vstack([Q] * 13 + [Q[:37]]).tocsr().astype(np.float32)
    Qbig.sort_indices()
    os.environ.pop("PB200_DEVICES", None)
    single = HNSW.load(folder)
    want = single.predict(Qbig, pred_params=HNSW.PredParams(efS=100, topk=10, threads=1), ret_csr=False)
    os.environ["PB200_DEVICES"] = "0,0,0"
    m = HNSW.load(folder)
    assert gpu_clib.clib_float32.pb200_hnsw_replicas(m.model_ptr) == 3
    got = m.predict(Qbig, pred_params=HNSW.PredParams(efS=100, topk=10, threads=1), ret_csr=False)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.uint32), want[1].view(np.uint32))


def test_bad_device_list_is_rejected(tmp_path, gpu_clib, devices_env):
    import subprocess
    import sys

    # the C layer aborts the process on errors (like the reference's exceptions through extern "C"): run in a child
    code = ("import os, sys; sys.path.insert(0, %r); os.environ['PB200_DEVICES'] = '0,99';\n"
            "from pecos_b200.hnsw import HNSW; HNSW.load(%r)" % (os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                                                                os.path.join(MID, "l2_dup")))
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode != 0 and "PB200_DEVICES" in r.stderr
