"""PairwiseANN limits that need no GPU: the dense width rule of pb200_pairwise_ann_dense_fits (ring depth switch at
d = 10,191 / 10,192, the widest searchable rows around 51,024 - 51,072) against the row layout of hnsw_host.h, the ValueError
a too-wide model raises before any native call, and the C restatement on NaN and infinite distances against the reference
library, which pins where the reference's heap sequence leaves a NaN."""
import numpy as np
import pytest
import scipy.sparse as smat

from tests.test_pairwise_ann_limits_gpu import assert_same_nan, dense_rule, nonfinite_case


def test_dense_fits_ring_depth_switch(clib):
    for d, depth in ((1, 4), (16, 4), (10191, 4), (10192, 0), (51024, 0)):
        fits, plan = clib.pairwise_ann_dense_fits(d)
        rule = dense_rule(d)
        assert fits and plan["stages"] == depth == rule[1], (d, plan)
        assert (plan["per_warp_bytes"], plan["vstride"]) == (rule[2], rule[3]), (d, plan, rule)
        assert plan["per_warp_bytes"] <= 200 * 1024


def test_dense_fits_exactly_the_row_layout_rule(clib):
    """Across 51,008 - 51,088 the widths that fit are exactly the ones dense_vstride leaves room for: every width up to
    51,024, then only multiples of 16 up to 51,072."""
    got = [d for d in range(51008, 51089) if clib.pairwise_ann_dense_fits(d)[0]]
    assert got == [d for d in range(51008, 51089) if dense_rule(d)[0]]
    assert got == list(range(51008, 51025)) + [51040, 51056, 51072]
    for d in range(51008, 51089):
        assert clib.pairwise_ann_dense_fits(d)[1]["vstride"] == dense_rule(d)[3]


@pytest.mark.parametrize("d", [51025, 51071, 51073])
def test_too_wide_dense_model_is_refused_in_python(clib, tmp_path, d):
    """Training and saving a wide model stay allowed (host-only, as in the reference); creating searchers and predicting raise
    ValueError naming the rule, before any native call (a plain object stands in for the searcher token)."""
    from pecos_b200.pairwise import PairwiseANN

    X = np.ones((3, d), np.float32)
    m = PairwiseANN.train(X, smat.eye(3, 2, dtype=np.float32, format="csc"))
    m.save(str(tmp_path / "wide"))
    with pytest.raises(ValueError, match="51,024.*51,072"):
        m.searchers_create(PairwiseANN.PredParams(batch_size=2, only_topk=2))
    fake = type("S", (), {"pred_params": PairwiseANN.PredParams(batch_size=2, only_topk=2)})()
    with pytest.raises(ValueError, match="feat_dim=%d" % d):
        m.predict(X[:2], np.array([0, 1], np.uint32), fake)
    # sparse models of any width stay searchable: only the dense query row is staged whole
    ms = PairwiseANN.train(smat.csr_matrix(X), smat.eye(3, 2, dtype=np.float32, format="csc"))
    ms._check_searchable()


def test_restatement_places_nan_like_the_reference_small(built, have_ref):
    """X = [[1], [nan], [2]], Q = [[-1]], one column of rows 0, 1, 2: the NaN stays where the heap sequence leaves it."""
    from oracle.pairwise import RefPairwise, oracle_predict

    X = np.array([[1], [np.nan], [2]], np.float32)
    Y = smat.csc_matrix(np.ones((3, 1), np.float32))
    Q = np.array([[-1]], np.float32)
    want = {1: ([0], [2.0]), 2: ([0, 1], [2.0, np.nan]), 3: ([0, 1, 2], [2.0, np.nan, 3.0])}
    for topk, (ids, dist) in want.items():
        I, M, D, V = oracle_predict(X, Y, Q, [0], topk)
        assert I[0].tolist() == ids and np.array_equal(D[0], np.array(dist, np.float32), equal_nan=True), topk
        if have_ref:
            assert_same_nan((I, M, D, V), RefPairwise.train(X, Y).predict(Q, [0], topk), f"topk={topk}")


@pytest.mark.parametrize("sparse", [False, True])
def test_restatement_on_nonfinite_columns_matches_reference(built, have_ref, sparse):
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    from oracle import restatement
    from oracle.pairwise import RefPairwise, oracle_predict

    if not sparse and restatement.host_isa() != 0:
        pytest.skip("the reference runs another SIMD clone here: NaN placement follows its own distance bits")
    X, Y, Q, keys = nonfinite_case(np.random.default_rng(70 + sparse), sparse)
    ref = RefPairwise.train(X, Y)
    for topk in (1, 2, 3, 10, 39, 40, 41, 127, 128, 129, 299, 300, 1024, 1025, 1100, 1101):
        for same in (False, True):
            assert_same_nan(oracle_predict(X, Y, Q, keys, topk, same), ref.predict(Q, keys, topk, same),
                            f"sparse={sparse} topk={topk} same={same}")
