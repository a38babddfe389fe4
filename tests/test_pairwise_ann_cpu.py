"""PairwiseANN checks that need no GPU: the C restatement of predict_single against the reference-recorded goldens and the
live reference library (ties included), the host-only writer and reader against the reference's save / load, and the overlay
of the seven pairwise_ann_fn_dict slots."""
import filecmp
import json
import os
import shutil
import subprocess
import sys
from ctypes import c_void_p

import numpy as np
import pytest
import scipy.sparse as smat

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden", "pairwise_ann")
CASES = ("dense_d70", "dense_d768", "sparse", "ties_dense", "ties_sparse", "same_input")
REFERENCE = "/root/reference"


def golden_case(name):
    from oracle.pairwise import read_c_model

    folder = os.path.join(GOLD, name)
    data_type = json.load(open(os.path.join(folder, "param.json")))["data_type"]
    X, Y = read_c_model(os.path.join(folder, "c_model"), data_type)
    Q = smat.load_npz(os.path.join(folder, "Q.npz")).tocsr() if data_type == "csr" else np.load(os.path.join(folder, "Q.npy"))
    return folder, data_type, X, Y, Q


def golden_runs(E, name):
    for key in E.files:
        parts = key.split("|")
        if parts[0] == name and len(parts) == 4 and parts[3] == "I":
            yield int(parts[1]), bool(int(parts[2]))


def assert_same(got, want):
    for tag, g, w in zip("IMDV", got, want):
        assert np.array_equal(np.asarray(g).view(np.uint32), np.asarray(w).view(np.uint32)), tag


@pytest.mark.parametrize("name", CASES)
def test_restatement_reproduces_goldens(built, name):
    from oracle.pairwise import oracle_predict

    E = np.load(os.path.join(GOLD, "expected.npz"))
    _, _, X, Y, Q = golden_case(name)
    keys = E[f"{name}|keys"]
    runs = list(golden_runs(E, name))
    assert len(runs) == 8
    for topk, same in runs:
        want = [E[f"{name}|{topk}|{int(same)}|{t}"] for t in "IMDV"]
        assert_same(oracle_predict(X, Y, Q, keys, topk, same), want)


def quantised_case(rng, sparse, N=300, L=25, d=37):
    if sparse:
        X = smat.csr_matrix((rng.integers(0, 3, size=(N, d)) * (rng.random((N, d)) < 0.1)).astype(np.float32))
        Q = smat.csr_matrix((rng.integers(0, 3, size=(40, d)) * (rng.random((40, d)) < 0.1)).astype(np.float32))
    else:
        X = rng.integers(-1, 2, size=(N, d)).astype(np.float32)
        Q = rng.integers(-1, 2, size=(40, d)).astype(np.float32)
    Y = smat.random(N, L, density=0.08, format="csc", dtype=np.float32, random_state=int(rng.integers(1 << 30)))
    Y.data = np.round(Y.data * 3 + 1).astype(np.float32)
    return X, Y, Q, rng.integers(0, L, size=40).astype(np.uint32)


@pytest.mark.parametrize("sparse", [False, True])
def test_restatement_matches_reference_live(built, have_ref, sparse):
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    from oracle.pairwise import RefPairwise, oracle_predict

    rng = np.random.default_rng(7 + sparse)
    X, Y, Q, keys = quantised_case(rng, sparse)
    ref = RefPairwise.train(X, Y)
    longest = int(np.diff(Y.indptr).max())
    for topk in (0, 1, 3, 10, longest, longest + 7):  # topk < n and topk >= n both occur
        for same in (False, True):
            assert_same(oracle_predict(X, Y, Q, keys, topk, same), ref.predict(Q, keys, topk, same))


@pytest.mark.parametrize("name", CASES)
def test_reference_saved_folders_pass_host_ingest(clib, name):
    folder, data_type, X, Y, _ = golden_case(name)
    info = clib.pairwise_ann_host_info(os.path.join(folder, "c_model"), data_type)
    assert (info["num_input_keys"], info["num_label_keys"], info["feat_dim"]) == (X.shape[0], Y.shape[1], X.shape[1])
    assert info["nnz_of_Y"] == Y.nnz and info["longest_column"] == int(np.diff(Y.indptr).max())
    with pytest.raises(ValueError):  # the other data type's pairwise_ann_t is refused
        clib.pairwise_ann_host_info(os.path.join(folder, "c_model"), "drm" if data_type == "csr" else "csr")


@pytest.mark.parametrize("name", CASES)
def test_save_matches_reference_save(clib, have_ref, tmp_path, name):
    """train + save here (host-only) vs the reference's own save of the same inputs; the folder loads in the reference with
    identical predictions.  config.json is byte-identical; index.mmap_store has the same blocks at the same offsets and differs
    at most in the zero padding after the last block and the metadata offset (DESIGN 4.8)."""
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    from oracle.pairwise import RefPairwise, read_c_model
    from oracle.restatement import read_mmap_store
    from pecos_b200.core import ScipyCscF32, ScipyCsrF32, ScipyDrmF32

    folder, data_type, X, Y, Q = golden_case(name)
    fd = clib.pairwise_ann_init(data_type, "ip")
    pX = ScipyCsrF32.init_from(X) if data_type == "csr" else ScipyDrmF32.init_from(np.ascontiguousarray(X))
    m = c_void_p(fd["train"](pX, ScipyCscF32.init_from(Y)))
    ours = str(tmp_path / "ours")
    fd["save"](m, ours.encode())
    fd["destruct"](m)
    theirs = os.path.join(folder, "c_model")
    assert filecmp.cmp(os.path.join(ours, "config.json"), os.path.join(theirs, "config.json"), shallow=False)
    a, b = read_mmap_store(os.path.join(ours, "index.mmap_store")), read_mmap_store(os.path.join(theirs, "index.mmap_store"))
    assert len(a) == len(b) and all(np.array_equal(x, y) for x, y in zip(a, b))
    ra = np.fromfile(os.path.join(ours, "index.mmap_store"), np.uint8)
    rb = np.fromfile(os.path.join(theirs, "index.mmap_store"), np.uint8)
    body = int(rb[-8:].view(np.uint64)[0])  # the reference's metadata offset = end of its last block
    assert np.array_equal(ra[:body], rb[:body]) and not ra[body:int(ra[-8:].view(np.uint64)[0])].any()
    keys = np.arange(Q.shape[0], dtype=np.uint32) % Y.shape[1]
    assert_same(RefPairwise.load(ours, data_type).predict(Q, keys, 10), RefPairwise.load(theirs, data_type).predict(Q, keys, 10))
    X2, Y2 = read_c_model(ours, data_type)
    assert (X2 != X).nnz == 0 if data_type == "csr" else np.array_equal(X2, X)


def test_python_validation_before_native_calls(clib):
    """Everything the reference validates, plus label keys, is refused in Python: no native call happens (none could: a
    searcher token needs a GPU, so a plain object stands in for it)."""
    from pecos_b200.pairwise import PairwiseANN

    X = np.ones((5, 3), np.float32)
    m = PairwiseANN.train(X, smat.eye(5, 4, dtype=np.float32, format="csr"))
    fake = type("S", (), {"pred_params": PairwiseANN.PredParams(batch_size=4, only_topk=2)})()
    with pytest.raises(ValueError):
        m.predict(X[:2], np.array([0, 4], np.uint32), fake)  # label key 4 >= num_label_keys 4
    with pytest.raises(ValueError):
        m.predict(X[:2], np.array([0, -1]), fake)
    with pytest.raises(ValueError):
        m.predict(X[:3], np.array([0, 1], np.uint32), fake)  # rows != batch
    with pytest.raises(ValueError):
        m.predict(np.ones((5, 2), np.float32), np.arange(5, dtype=np.uint32), fake)  # feat_dim
    with pytest.raises(ValueError):
        m.predict(smat.csr_matrix(X), np.arange(5, dtype=np.uint32), fake)  # data type
    with pytest.raises(TypeError):
        m.predict(X[:2], [0, 1], fake)
    with pytest.raises(ValueError):
        m.predict(X, np.arange(5, dtype=np.uint32) % 4, fake)  # batch > batch_size
    with pytest.raises(ValueError):
        PairwiseANN.train(X, np.eye(5, dtype=np.float32))
    with pytest.raises(ValueError):
        PairwiseANN.train(X[:4], smat.eye(5, 4, dtype=np.float32, format="csc"))


def test_overlay_swaps_all_seven_pairwise_slots(tmp_path, built, have_ref):
    if not os.path.isdir(os.path.join(REFERENCE, "pecos")):
        pytest.skip("the reference checkout is not on this box")
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    scratch = str(tmp_path / "refpy")
    shutil.copytree(os.path.join(REFERENCE, "pecos"), os.path.join(scratch, "pecos"))
    subprocess.run(["chmod", "-R", "u+w", scratch], check=True)
    shutil.copy(os.path.join(ROOT, "oracle", "_ref", "libpecos_float32.so"), os.path.join(scratch, "pecos", "core", "libpecos_float32.so"))
    p = os.path.join(scratch, "pecos", "utils", "smat_util.py")
    src = open(p).read().replace("smat.sputils.get_index_dtype", "smat._sputils.get_index_dtype").replace("copy=False", "copy=None")
    open(p, "w").write(src)
    code = r"""
import sys, ctypes, json
sys.path.insert(0, %r); sys.path.insert(0, %r)
from pecos.core import clib
from pecos_b200 import integration
before = {k: {s: (f.restype, tuple(f.argtypes or ())) for s, f in d.items() if hasattr(f, "argtypes")} for k, d in clib.pairwise_ann_fn_dict.items()}
names = integration.overlay(clib, require_gpu=False)
def where(fn):
    class I(ctypes.Structure):
        _fields_ = [("f", ctypes.c_char_p), ("b", ctypes.c_void_p), ("s", ctypes.c_char_p), ("a", ctypes.c_void_p)]
    dl = ctypes.CDLL(None); dl.dladdr.argtypes = [ctypes.c_void_p, ctypes.POINTER(I)]
    i = I(); dl.dladdr(ctypes.cast(fn, ctypes.c_void_p).value, ctypes.byref(i)); return i.f.decode()
out = {"swapped": names}
out["pairwise"] = {"%%s_%%s" %% (k[0], s): where(f) for k, d in clib.pairwise_ann_fn_dict.items() for s, f in d.items() if hasattr(f, "argtypes")}
out["protos_kept"] = all((f.restype, tuple(f.argtypes or ())) == before[k][s] for k, d in clib.pairwise_ann_fn_dict.items() for s, f in d.items() if hasattr(f, "argtypes"))
out["other"] = {n: where(getattr(clib.clib_float32, n)) for n in ("c_sparse_matmul_csc_f32", "c_ann_hnsw_train_drm_ip_f32")}
print("RESULT" + json.dumps(out))
""" % (scratch, ROOT)
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    out = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT")][0][6:])
    assert len(out["pairwise"]) == 14, out["pairwise"]
    assert all(p.endswith("libpecos_b200_float32.so") for p in out["pairwise"].values()), out["pairwise"]
    assert out["protos_kept"]
    assert all(p.endswith("libpecos_float32.so") for p in out["other"].values()), out["other"]
    assert sum(n.startswith("c_pairwise_ann_") for n in out["swapped"]) == 14
