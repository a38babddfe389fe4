"""CPU tests of HNSW search with NaN and infinite distances (the GPU side is tests/test_hnsw_nonfinite_gpu.py):

* the C restatement the GPU kernel is compared with bit for bit is pinned to the reference library (oracle/_ref) on the
  non-finite indices and queries of tests/hnsw_nonfinite_util.py -- ids and distance bits equal, two NaNs of any payload
  equal -- and on one index the reference trained with the non-finite rows included; every result also meets a float64
  evaluation of the returned (query, id) pairs;
* the restatement reproduces the reference outputs recorded in tests/golden/hnsw_nonfinite;
* the dense width rule of the search plan (pb200_hnsw_dense_plan, host-only) equals its restatement in Python over a sweep of
  widths, neighbour-list lengths, ring depth settings and ef.
"""
import json
import os

import numpy as np
import pytest
import scipy.sparse as smat

from . import hnsw_nonfinite_util as nf

HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden", "hnsw_nonfinite")
GRID = [(10, 10), (64, 10), (5, 40), (512, 10), (513, 10), (600, 100)]
WARP_SMEM_MAX = 200 * 1024
EF_SMEM_MAX = 512


def _ref_index(folder, X, metric, edits, M=12, efC=40):
    """Reference-trained index of the finite rows X with `edits` (dict, or a function of the parsed index) written into the
    saved file: (restatement, reference handle of the saved file, rows as searched)."""
    from oracle import ref, restatement

    from .util import save_hnsw_index

    save_hnsw_index(folder, X, M, efC, metric, True, threads=1)
    if callable(edits):
        edits = edits(restatement.OracleHNSW(folder))
    nf.overwrite_values(folder, edits)
    sparse = smat.issparse(X)
    r = ref.RefHNSW.load(os.path.join(folder, "c_model"), metric, data_type="csr" if sparse else "drm")
    return restatement.OracleHNSW(folder, isa=restatement.host_isa()), r, (nf.apply_sparse(X, edits) if sparse else nf.apply_dense(X, edits))


def _compare(o, r, X, Q, metric, skip, what):
    for efS, topk in GRID:
        oi, od = o.predict(Q, efS, topk)
        ri, rd = r.predict(Q, efS, topk, threads=1)
        nf.assert_same_nan_hnsw((oi, od), (ri, rd), f"restatement vs reference {what} efS={efS} topk={topk}")
        nf.f64_check(X, Q, metric, oi, od, skip, what)


@pytest.mark.parametrize("variant,metric", [("scattered", "ip"), ("scattered", "l2"), ("entry_nan", "ip"), ("entry_neginf", "ip")])
@pytest.mark.parametrize("d", [17, 70, 768])
def test_dense_restatement_equals_reference(built, have_ref, tmp_path, d, variant, metric):
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    from oracle import restatement

    if restatement.host_isa() != 0:
        pytest.skip("the reference runs another SIMD clone on this CPU: the order-dependent row differs by design")
    rng = np.random.default_rng(1000 * d + (metric == "l2"))
    X = nf.dense_rows(rng, 600, d)
    kinds = {}

    def edits(oo):
        e, k = nf.dense_edits(oo, d, metric, variant)
        kinds.update(k)
        return e

    o, r, Xs = _ref_index(str(tmp_path / "i"), X, metric, edits)
    Q, order_q = nf.dense_queries(rng, d)
    skip = {(order_q, n) for n, k in kinds.items() if k == "order"} if (order_q is not None and metric == "ip") else set()
    _compare(o, r, Xs, Q, metric, skip, f"d={d} {variant} {metric}")


@pytest.mark.parametrize("metric", ["ip", "l2"])
def test_sparse_restatement_equals_reference(built, have_ref, tmp_path, metric):
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    rng = np.random.default_rng(7 + (metric == "l2"))
    X = nf.sparse_rows(rng, 600)
    o, r, Xs = _ref_index(str(tmp_path / "i"), X, metric, nf.sparse_edits(X, 3))
    _compare(o, r, Xs, nf.sparse_queries(rng), metric, (), f"csr {metric}")


def test_index_trained_with_nonfinite_rows(built, have_ref, tmp_path):
    """The reference's own builder on rows that already hold NaN and +-1e20 (its graph then follows NaN comparisons too)."""
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    from oracle import ref, restatement

    if restatement.host_isa() != 0:
        pytest.skip("the reference runs another SIMD clone on this CPU")
    rng = np.random.default_rng(77)
    d = 70
    X = nf.dense_rows(rng, 500, d)
    sp = nf.spots(d)
    for i, n in enumerate(range(10, 60, 5)):
        X[n, sp[i % len(sp)]] = (np.nan, nf.BIG, -nf.BIG)[i % 3]
    folder = str(tmp_path / "i")
    from .util import save_hnsw_index

    save_hnsw_index(folder, X, 12, 40, "ip", True, threads=1)
    r = ref.RefHNSW.load(os.path.join(folder, "c_model"), "ip")
    o = restatement.OracleHNSW(folder, isa=0)
    assert np.array_equal(o.vectors().view(np.uint32), X.view(np.uint32))
    Q, order_q = nf.dense_queries(rng, d)
    _compare(o, r, X, Q, "ip", set(), "trained with non-finite rows")


def test_restatement_reproduces_recorded_reference_outputs(built):
    from oracle import restatement

    E = np.load(os.path.join(GOLD, "expected.npz"))
    index = json.load(open(os.path.join(GOLD, "expected_index.json")))
    models, classes = {}, set()
    for it in index:
        folder = os.path.join(GOLD, it["model"])
        if it["model"] not in models:
            q = os.path.join(folder, "Q.npz")
            Q = smat.load_npz(q).tocsr() if os.path.exists(q) else np.load(os.path.join(folder, "Q.npy"))
            models[it["model"]] = (restatement.OracleHNSW(folder, isa=0), Q)
        o, Q = models[it["model"]]
        got = o.predict(Q, it["efS"], it["topk"])
        want = (E[it["key"] + "|idx"], E[it["key"] + "|dist"])
        nf.assert_same_nan_hnsw(got, want, it["key"])
        classes |= {"nan"} if np.isnan(want[1]).any() else set()
        classes |= {"+inf"} if (want[1] == np.inf).any() else set()
        classes |= {"-inf"} if (want[1] == -np.inf).any() else set()
    assert set(models) == {"dense_ip_d70", "dense_l2_d70", "sparse_ip"} and classes == {"nan", "+inf", "-inf"}


# ------------------------------------------------------------------------------------------------------ the width rule
def dense_plan_rule(d, max_degree, stages, ef):
    """(fits, ring depth, heap in shared memory, per-warp bytes) of a dense search, restated from hnsw_engine.h: the heap in
    shared memory (ef <= 512 only) at depths stages, 4, 0, then the heap in global memory at the same depths; the first
    slice [query | ring rows | mbarriers | nbmax ids + distances | heap] of at most 204,800 bytes wins."""
    vstride = 64 * ((d // 16 + 3) // 4) + (16 if d % 16 else 0)
    nbmax = (max_degree + 31) // 32 * 32
    first = 0 if stages <= 0 else (4 if stages <= 4 else 8)
    depths = [s for s in (8, 4, 0) if s <= first]
    per_warp = None
    for in_smem in ([True] if ef <= EF_SMEM_MAX else []) + [False]:
        for s in depths:
            heap = (ef + 1) * 8 if in_smem else 0
            per_warp = (vstride * 4 * (1 + s) + 8 * s + nbmax * 8 + heap + 15) & ~15
            if per_warp <= WARP_SMEM_MAX:
                return True, s, in_smem, per_warp
    return False, 0, False, per_warp


def test_dense_width_rule_matches_the_engine_plan(clib):
    widths = sorted(set(list(range(1, 200)) + list(range(1000, 60000, 997)) + [10176, 10129, 12288] +
                        [w + o for w in (50063, 50880, 50895, 50959, 51008, 51087, 51136) for o in (-1, 0, 1, 2)]))
    n = 0
    for M in (8, 16, 48, 64):
        for stages in (0, 4, 8):
            for ef in (10, 100, 512, 513, 1000):
                for d in widths:
                    fits, plan = clib.hnsw_dense_plan(d, 2 * M, stages, ef, 1)
                    want = dense_plan_rule(d, 2 * M, stages, ef)
                    assert fits == want[0], (M, stages, ef, d, plan, want)
                    if fits:
                        assert (plan["stages"], bool(plan["heap_in_smem"]), plan["per_warp_bytes"]) == want[1:], (M, stages, ef, d)
                    n += 1
    assert n > 10000
    # the limit depends on (d, M) only: with M = 16 every ef serves d up to 51,087, and every multiple of 16 up to 51,136
    for ef in (10, 100, 512, 513, 1000):
        assert clib.hnsw_dense_plan(51087, 32, 4, ef, 1)[0] and not clib.hnsw_dense_plan(51089, 32, 4, ef, 1)[0]
        assert clib.hnsw_dense_plan(51136, 32, 4, ef, 1)[0] and not clib.hnsw_dense_plan(51152, 32, 4, ef, 1)[0]
        assert clib.hnsw_dense_plan(50959, 96, 4, ef, 1)[0] and not clib.hnsw_dense_plan(50961, 96, 4, ef, 1)[0]
        assert clib.hnsw_dense_plan(51008, 96, 4, ef, 1)[0] and not clib.hnsw_dense_plan(51024, 96, 4, ef, 1)[0]
    # where the heap must leave shared memory at ef <= 512: d = 50,500 at ef = 512 (it stays there at ef = 100)
    assert clib.hnsw_dense_plan(50500, 32, 4, 512, 10)[1]["heap_in_smem"] == 0
    assert clib.hnsw_dense_plan(50500, 32, 4, 100, 10)[1]["heap_in_smem"] == 1
    # the order 8 -> 4 -> 0 with the heap in shared memory comes first: d = 10,176 runs depth 0 at ef = 512
    assert clib.hnsw_dense_plan(10176, 32, 4, 512, 10)[1]["stages"] == 0


def test_shard_key_puts_every_nan_last():
    """The key rule of the exchange records (hnsw_shard_util): NaN of either sign and any payload after +inf, ties by slot."""
    from .hnsw_shard_util import hnsw_shard_records
    from .util import merge_shards_numpy

    bits = np.array([0x7FC00000, 0xFFC00000, 0x7F800000, 0x3F800000, 0xFF800000, 0x7FFFFFFF, 0xFFFFFFFF, 0x80000000], np.uint32)
    dist = bits.view(np.float32)[None, :]
    idx = np.arange(8, dtype=np.uint32)[None, :]
    keys, ids, vals = hnsw_shard_records(idx, dist, np.array([8]), 0, 0, 8)
    out, _, _ = merge_shards_numpy(keys[None], ids[None], vals[None], np.array([[8]]), 8)
    assert out[0].tolist() == [4, 7, 3, 2, 0, 1, 5, 6]
