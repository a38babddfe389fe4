"""PairwiseANN on the GPU: I / M / D / V bit-identical to the reference-recorded goldens, to the C restatement and to the live
reference library (oracle/_ref) on random dense and sparse inputs -- long columns (split over many work items, global-memory
replay), heavy ties (replay path taken), tie-free inputs (replay never taken), is_same_input, empty columns and topk from 0
to beyond the longest column -- plus the reference's test_pairwise_ann.py scenarios, save / load in both directions and
concurrent searcher tokens."""
import os
import threading

import numpy as np
import pytest
import scipy.sparse as smat

from tests.test_pairwise_ann_cpu import CASES, GOLD, assert_same, golden_case, golden_runs

pytestmark = pytest.mark.gpu


def _pp(bsz, topk):
    from pecos_b200.pairwise import PairwiseANN

    return PairwiseANN.PredParams(batch_size=max(bsz, 1), only_topk=topk)


def gpu_predict(model, Q, keys, topk, same=False):
    s = model.searchers_create(_pp(len(keys), topk))
    out = [a.copy() for a in model.predict(Q, keys, s, is_same_input=same)]
    return out, s.counters()


@pytest.mark.parametrize("name", CASES)
def test_goldens(gpu_clib, name):
    from pecos_b200.pairwise import PairwiseANN

    E = np.load(os.path.join(GOLD, "expected.npz"))
    folder, _, _, _, Q = golden_case(name)
    m = PairwiseANN.load(folder)
    keys = E[f"{name}|keys"]
    for topk, same in golden_runs(E, name):
        want = [E[f"{name}|{topk}|{int(same)}|{t}"] for t in "IMDV"]
        got, _ = gpu_predict(m, Q, keys, topk, same)
        assert_same(got, want)


def _random_case(rng, sparse, N, L, d, levels, long_col=0, empty_cols=2):
    if sparse:
        dens = rng.random((N, d)) < 0.05
        vals = rng.integers(1, levels + 1, size=(N, d)) if levels else rng.random((N, d)) + 0.1
        X = smat.csr_matrix((vals * dens).astype(np.float32))
    else:
        X = (rng.integers(-levels, levels + 1, size=(N, d)) if levels else rng.standard_normal((N, d))).astype(np.float32)
    rows, cols = [], []
    p = 1.0 / np.arange(1, L + 1) ** 1.2
    p[:empty_cols] = 0
    p /= p.sum()
    for r in range(N):
        for c in rng.choice(L, size=2, replace=False, p=p):
            rows.append(r); cols.append(c)  # noqa: E702
    if long_col:
        rows += list(rng.choice(N, size=long_col, replace=False)); cols += [L - 1] * long_col  # noqa: E702
    data = (rng.integers(1, 5, size=len(rows)) / 2).astype(np.float32)
    Y = smat.csc_matrix((data, (rows, cols)), shape=(N, L))
    Y.sum_duplicates()
    return X, Y


def _queries(rng, X, nq, levels):
    if isinstance(X, smat.csr_matrix):
        dens = rng.random((nq, X.shape[1])) < 0.05
        vals = rng.integers(1, levels + 1, size=dens.shape) if levels else rng.random(dens.shape) + 0.1
        return smat.csr_matrix((vals * dens).astype(np.float32))
    return (rng.integers(-levels, levels + 1, size=(nq, X.shape[1])) if levels else rng.standard_normal((nq, X.shape[1]))).astype(np.float32)


@pytest.mark.parametrize("sparse", [False, True])
@pytest.mark.parametrize("levels", [0, 1])
def test_random_against_reference_and_restatement(gpu_clib, have_ref, sparse, levels):
    """levels = 1: values in {-1, 0, 1} (dense) or {0, 1} (sparse) -- ties everywhere, the replay path must run.
    levels = 0: continuous values -- dense top-10s are tie-free and never replay (sparse rows disjoint from the query tie at
    exactly 1.0, and a 50,000-entry column sorted in full can hold equal floats).  The last column holds >= 50,000 entries."""
    from oracle.pairwise import RefPairwise, oracle_predict
    from pecos_b200.pairwise import PairwiseANN

    rng = np.random.default_rng(100 + 2 * sparse + levels)
    N, L, d = 64000, 64, (96 if sparse else 70)
    X, Y = _random_case(rng, sparse, N, L, d, levels, long_col=50000 if not levels else 60000)
    assert np.diff(Y.indptr).max() >= 50000 and np.diff(Y.indptr).min() == 0
    nq = 96
    Q = _queries(rng, X, nq, levels)
    keys = np.concatenate([[L - 1, 0, 1], rng.integers(0, L, size=nq - 3)]).astype(np.uint32)
    m = PairwiseANN.train(X, Y)
    ref = RefPairwise.train(X, Y) if have_ref else None
    for topk in (0, 1, 10, 1000, 70000):
        for same in (False, True):
            got, cnt = gpu_predict(m, Q, keys, topk, same)
            want = oracle_predict(X, Y, Q, keys, topk, same)
            assert_same(got, want)
            if ref is not None:
                assert_same(got, ref.predict(Q, keys, topk, same, threads=8))
            if topk:
                assert cnt["pairs"] == nq and cnt["distances"] == int(np.diff(Y.indptr)[keys].sum())
                if levels:
                    assert cnt["replays"] > 0
                elif topk <= 10 and not sparse:
                    assert cnt["replays"] == 0, cnt


def test_reference_scenarios(gpu_clib, tmp_path):
    """test/pecos/ann/test_pairwise_ann.py: save_and_load, consistency between drm and csr, predict with same input."""
    from pecos_b200.pairwise import PairwiseANN

    rng = np.random.default_rng(3)
    # test_save_and_load
    N, D, bsz, k = 10000, 64, 250, 10
    X = rng.standard_normal((N, D)).astype(np.float32)
    Y = smat.eye(N, dtype=np.float32, format="csc")
    keys = np.arange(bsz).astype(np.uint32)
    m = PairwiseANN.train(X, Y, train_params=PairwiseANN.TrainParams(metric_type="ip"))
    s = m.searchers_create(pred_params=_pp(bsz, k), num_searcher=1)
    It, Mt, Dt, Vt = [a.copy() for a in m.predict(X[:bsz], keys, s)]
    m.save(str(tmp_path / "pw"))
    del m, s
    m = PairwiseANN.load(str(tmp_path / "pw"), lazy_load=True)
    s = m.searchers_create(pred_params=_pp(bsz, k), num_searcher=2)
    assert_same(m.predict(X[:bsz], keys, s), (It, Mt, Dt, Vt))
    # test_consistency_between_drm_and_csr
    N = D = 128
    X = rng.standard_normal((N, D)).astype(np.float32)
    Y = smat.eye(N, dtype=np.float32, format="csc")
    keys = np.arange(3).astype(np.uint32)
    md, ms = PairwiseANN.train(X, Y), PairwiseANN.train(smat.csr_matrix(X), Y)
    Id, Md, Dd, Vd = md.predict(X[:3], keys, md.searchers_create(_pp(3, 2)))
    Is, Ms, Ds, Vs = ms.predict(smat.csr_matrix(X[:3]), keys, ms.searchers_create(_pp(3, 2)))
    assert np.array_equal(Id, [[0, 0], [1, 0], [2, 0]]) and np.array_equal(Md, [[1, 0], [1, 0], [1, 0]])
    assert np.array_equal(Vd, [[1, 0], [1, 0], [1, 0]])
    assert np.array_equal(Id, Is) and np.array_equal(Md, Ms) and np.array_equal(Vd, Vs) and np.allclose(Dd, Ds, atol=1e-4)
    # test_predict_with_same_input
    X = np.array([[1, 0], [2, 0], [3, 0], [4, 0], [5, 0]], dtype=np.float32)
    Y = smat.csr_matrix(np.array([[1.1, 0, 0, 0], [2.1, 2.2, 0, 0], [0, 3.2, 3.3, 0], [0, 0, 4.3, 4.4], [0, 0, 0, 5.4]], dtype=np.float32))
    m = PairwiseANN.train(X, Y)
    I, M, Dm, V = m.predict(X[:4], np.arange(4).astype(np.uint32), m.searchers_create(_pp(4, 3)))
    assert np.array_equal(I, [[1, 0, 0], [2, 1, 0], [3, 2, 0], [4, 3, 0]])
    assert np.array_equal(M, [[1, 1, 0], [1, 1, 0], [1, 1, 0], [1, 1, 0]])
    assert np.array_equal(Dm, [[-1, 0, 0], [-5, -3, 0], [-11, -8, 0], [-19, -15, 0]])
    assert np.allclose(V, [[2.1, 1.1, 0], [3.2, 2.2, 0], [4.3, 3.3, 0], [5.4, 4.4, 0]], atol=1e-6)


@pytest.mark.parametrize("name", ["dense_d70", "sparse", "ties_sparse"])
def test_save_load_both_directions(gpu_clib, have_ref, tmp_path, name):
    """a folder saved here loads in the reference, a reference-saved folder loads here: same outputs everywhere."""
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    from oracle.pairwise import RefPairwise
    from pecos_b200.pairwise import PairwiseANN

    folder, data_type, X, Y, Q = golden_case(name)
    keys = np.arange(Q.shape[0], dtype=np.uint32) % Y.shape[1]
    ours = PairwiseANN.train(X, Y)
    ours.save(str(tmp_path / "ours"))
    want = RefPairwise.load(os.path.join(folder, "c_model"), data_type).predict(Q, keys, 10)
    assert_same(RefPairwise.load(str(tmp_path / "ours" / "c_model"), data_type).predict(Q, keys, 10), want)
    assert_same(gpu_predict(PairwiseANN.load(folder), Q, keys, 10)[0], want)
    assert_same(gpu_predict(PairwiseANN.load(str(tmp_path / "ours")), Q, keys, 10)[0], want)


def test_two_tokens_from_two_threads(gpu_clib):
    from pecos_b200.pairwise import PairwiseANN

    rng = np.random.default_rng(11)
    X, Y = _random_case(rng, False, 25000, 40, 70, 1, long_col=20000)
    Q = _queries(rng, X, 200, 1)
    keys = rng.integers(0, 40, size=200).astype(np.uint32)
    m = PairwiseANN.train(X, Y)
    serial = [gpu_predict(m, Q, keys, t)[0] for t in (5, 50)]
    toks = [m.searchers_create(_pp(200, t)) for t in (5, 50)]
    res = [None, None]

    def run(i):
        for _ in range(5):
            res[i] = [a.copy() for a in m.predict(Q, keys, toks[i])]

    th = [threading.Thread(target=run, args=(i,)) for i in range(2)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert_same(res[0], serial[0])
    assert_same(res[1], serial[1])


def test_out_of_range_label_key_raises_before_native_call(gpu_clib):
    from pecos_b200.pairwise import PairwiseANN

    X = np.ones((5, 3), np.float32)
    m = PairwiseANN.train(X, smat.eye(5, 4, dtype=np.float32, format="csc"))
    s = m.searchers_create(_pp(2, 2))
    s.Imat[:] = 77
    with pytest.raises(ValueError):
        m.predict(X[:2], np.array([1, 4], np.uint32), s)
    assert (s.Imat == 77).all()  # nothing was reset or written: the call never reached the library
