"""GPU tests of HNSW search with NaN and infinite distances: dense (ip, l2; d = 17, 70, 768: main chunks, 4-wide remainder and
scalar tail; ring depths 0, 4, 8) and sparse (ip, l2), index sharding, the resident path and the whole-graph walk a NaN upper
bound causes (with the candidate-queue retry and the full bitmap clear).

Indices are built from finite rows and then get chosen stored values overwritten (tests/hnsw_nonfinite_util.py), so the graph
is the finite one and only distances change.  Every search is checked three ways:
* against the C restatement (oracle/restatement.py, avx512f order): ids exact, distance bits exact with two NaNs of any payload
  equal (the GPU returns 0x7FFFFFFF for every NaN, x86 the first NaN operand or 0xFFC00000; payloads are not matched), and the
  counters (distances, expansions, hops, queries) equal -- the walk itself is the reference's, not just the answer;
* against the reference library where oracle/_ref is built (same bar when it runs the avx512f clone or the index is sparse;
  else without the query whose class depends on the lane order, and ids equal with distances allclose, NaN = NaN), and
  always against the reference outputs recorded in tests/golden/hnsw_nonfinite;
* against a float64 evaluation of every returned (query, id): finite distances within the float32 accumulation bound, the
  forced classes (NaN, +inf, -inf) exactly.  This one is independent of both C implementations.
"""
import json
import os

import numpy as np
import pytest
import scipy.sparse as smat

from . import hnsw_nonfinite_util as nf
from .util import save_hnsw_index

pytestmark = pytest.mark.gpu

GRID = [(10, 10), (64, 10), (5, 40), (512, 10), (513, 10), (600, 100)]
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hnsw_nonfinite")


def counters(m):
    from ctypes import c_uint64

    from pecos_b200.core import get_clib

    out = (c_uint64 * 4)()
    get_clib().clib_float32.pb200_hnsw_get_counters(m.model_ptr, out)
    return [int(v) for v in out]


class _Case(object):
    """One index with overwritten rows, searched by the engine, the restatement and (where trained by it) the reference."""

    def __init__(self, folder, X, metric, have_ref, edits, M=12, efC=40):
        from oracle import restatement
        from pecos_b200.hnsw import HNSW

        self.sparse, self.metric = smat.issparse(X), metric
        r = save_hnsw_index(folder, X, M, efC, metric, have_ref)
        if callable(edits):
            edits = edits(restatement.OracleHNSW(folder))
        nf.overwrite_values(folder, edits)
        self.X = nf.apply_sparse(X, edits) if self.sparse else nf.apply_dense(X, edits)
        self.ref = None
        if r is not None:
            from oracle import ref

            self.ref = ref.RefHNSW.load(os.path.join(folder, "c_model"), metric, data_type="csr" if self.sparse else "drm")
        self.m = HNSW.load(folder)
        self.o = restatement.OracleHNSW(folder, isa=0)
        self.isa = restatement.host_isa()
        assert np.array_equal(np.isnan(self.o.vectors().toarray() if self.sparse else self.o.vectors()),
                              np.isnan(self.X.toarray() if self.sparse else self.X))
        self.want = {}
        self.seen = set()

    def check(self, Q, efS, topk, skip=(), order_q=None, what=""):
        from pecos_b200.hnsw import HNSW

        key = (id(Q), efS, topk)
        if key not in self.want:
            oi, od, oc = self.o.predict(Q, efS, topk, return_counters=True)
            if self.ref is not None:
                ri, rd = self.ref.predict(Q, efS, topk, threads=1)
                if self.sparse or self.isa == 0:
                    nf.assert_same_nan_hnsw((ri, rd), (oi, od), f"restatement vs reference {what} efS={efS} topk={topk}")
                else:  # another SIMD clone: the order-dependent query differs by design, the rest in the last bits
                    keep = np.array([q != order_q for q in range(Q.shape[0])])
                    assert np.mean(ri[keep] == oi[keep]) > 0.99
                    assert np.allclose(rd[keep], od[keep], rtol=1e-5, atol=1e-6, equal_nan=True)
            self.want[key] = (oi, od, [int(oc[:, 0].sum()), int(oc[:, 1].sum()), int(oc[:, 2].sum()), Q.shape[0]])
        oi, od, oc = self.want[key]
        gi, gd = self.m.predict(Q, pred_params=HNSW.PredParams(efS=efS, topk=topk), ret_csr=False)
        nf.assert_same_nan_hnsw((gi, gd), (oi, od), f"engine vs restatement {what} efS={efS} topk={topk}")
        assert counters(self.m) == oc, f"counters {what} efS={efS} topk={topk}"
        assert nf.f64_check(self.X, Q, self.metric, gi, gd, skip, what) > 0
        self.seen |= {"nan"} if np.isnan(gd).any() else set()
        self.seen |= {"+inf"} if (gd == np.inf).any() else set()
        self.seen |= {"-inf"} if (gd == -np.inf).any() else set()
        return gi, gd


def dense_case(tmp_path, have_ref, d, metric, variant, seed=0, N=1000):
    rng = np.random.default_rng(1000 * d + 10 * seed + (metric == "l2"))
    X = nf.dense_rows(rng, N, d)
    kinds = {}

    def edits(o):
        e, k = nf.dense_edits(o, d, metric, variant)
        kinds.update(k)
        return e

    c = _Case(str(tmp_path / f"{variant}_{metric}_{d}"), X, metric, have_ref, edits)
    Q, order_q = nf.dense_queries(rng, d)
    skip = {(order_q, n) for n, k in kinds.items() if k == "order"} if (order_q is not None and metric == "ip") else set()
    return c, Q, skip, order_q, kinds


VARIANTS = [("scattered", "ip"), ("scattered", "l2"), ("entry_nan", "ip"), ("entry_nan", "l2"), ("entry_neginf", "ip")]


@pytest.mark.parametrize("variant,metric", VARIANTS)
@pytest.mark.parametrize("d", [17, 70, 768])
def test_dense_nonfinite_rows_and_queries(tmp_path, gpu_clib, have_ref, d, variant, metric):
    c, Q, skip, order_q, _ = dense_case(tmp_path, have_ref, d, metric, variant)
    for stages in (0, 4, 8):
        assert gpu_clib.clib_float32.pb200_hnsw_set_stages(c.m.model_ptr, stages) == stages
        for efS, topk in GRID:
            c.check(Q, efS, topk, skip, order_q, f"d={d} {variant} stages={stages}")
    want = {"scattered": {"nan", "+inf"} | ({"-inf"} if metric == "ip" else set()), "entry_nan": {"nan"},
            "entry_neginf": {"-inf", "nan"}}[variant]
    assert want <= c.seen, (variant, c.seen)


def test_order_dependent_row_is_nan_in_lane_order(tmp_path, gpu_clib, have_ref):
    """The row with two +1.8e38 products in one SIMD lane and two -1.8e38 in another: NaN for the query that meets it, as the
    avx512 lane order gives, though its float64 (and left-to-right) sum is 0."""
    c, Q, skip, order_q, kinds = dense_case(tmp_path, have_ref, 70, "ip", "scattered")
    rows = [n for n, k in kinds.items() if k == "order"]
    gi, gd = c.check(Q[order_q:order_q + 1], 1000, 1000, {(0, n) for n in rows}, 0)  # every reachable node
    hit = [j for j in range(gi.shape[1]) if int(gi[0, j]) in rows]
    assert hit and all(np.isnan(gd[0, j]) for j in hit)
    assert float(np.float32(nf.HALF_LANE) * nf.BIG) * 2 > nf.FLT_MAX > float(np.float32(nf.HALF_LANE) * nf.BIG)


@pytest.mark.parametrize("metric", ["ip", "l2"])
def test_sparse_nonfinite_rows_and_queries(tmp_path, gpu_clib, have_ref, metric):
    """NaN on a matched and on an unmatched index, overflowing products, inf x a stored 0.0 and a 5,000-entry query (searched
    in global memory) carrying a NaN; the reference's sparse "l2" is -2<x,y>."""
    rng = np.random.default_rng(7 + (metric == "l2"))
    X = nf.sparse_rows(rng, 1200)
    c = _Case(str(tmp_path / metric), X, metric, have_ref, nf.sparse_edits(X, 3))
    Q = nf.sparse_queries(rng)
    assert np.diff(Q.indptr).max() > 4096
    for efS, topk in GRID + [(1300, 1300)]:  # the last returns every reachable node: +inf distances come last
        c.check(Q, efS, topk, what=f"csr {metric}")
    assert {"nan", "+inf", "-inf"} <= c.seen


def test_whole_graph_walk_with_small_and_default_queue(tmp_path, gpu_clib, have_ref, monkeypatch):
    """A NaN at the entry node keeps the upper bound NaN, so no candidate is ever cut off: every query walks until its
    candidate queue is empty (ef expansions, distances to nearly the whole graph).  With a 64-entry
    candidate queue the batch overflows and is re-run (and the visited bitmap is cleared in full); the default capacity gives
    the same ids, bits and counters."""
    from pecos_b200.hnsw import HNSW

    c, Q, skip, order_q, _ = dense_case(tmp_path, have_ref, 70, "l2", "entry_nan")
    folder = str(tmp_path / "entry_nan_l2_70")
    monkeypatch.setenv("PB200_HNSW_VCAP", "64")
    small = HNSW.load(folder)
    pp = HNSW.PredParams(efS=600, topk=100)
    a = small.predict(Q, pred_params=pp, ret_csr=False)
    ca = counters(small)
    assert gpu_clib.clib_float32.pb200_hnsw_vcap_retries(small.model_ptr) > 0
    monkeypatch.delenv("PB200_HNSW_VCAP")
    b = c.check(Q, 600, 100, skip, order_q, "default queue")
    assert gpu_clib.clib_float32.pb200_hnsw_vcap_retries(c.m.model_ptr) == 0
    nf.assert_same_nan_hnsw(a, b, "queue of 64 vs default")
    assert ca == counters(c.m)
    # with a NaN upper bound no candidate is ever cut off: each query expands exactly the ef nodes its result heap admitted
    assert ca[1] == Q.shape[0] * 600


@pytest.mark.parametrize("sparse", [False, True])
def test_resident_batch_equals_host_buffer_search(tmp_path, gpu_clib, have_ref, sparse):
    from ctypes import POINTER, byref, c_float, c_uint32

    from pecos_b200.hnsw import HNSW

    if sparse:
        rng = np.random.default_rng(9)
        X = nf.sparse_rows(rng, 800)
        c = _Case(str(tmp_path / "sp"), X, "ip", have_ref, nf.sparse_edits(X, 4))
        Q = nf.sparse_queries(rng)
    else:
        c, Q, _, _, _ = dense_case(tmp_path, have_ref, 70, "ip", "scattered", seed=1)
    lib = gpu_clib.clib_float32
    view, kind = HNSW.create_pymat(Q)
    (lib.pb200_hnsw_resident_upload_csr if sparse else lib.pb200_hnsw_resident_upload)(c.m.model_ptr, byref(view))
    for efS, topk in GRID:
        want = c.m.predict(Q, pred_params=HNSW.PredParams(efS=efS, topk=topk), ret_csr=False)
        lib.pb200_hnsw_resident_predict(c.m.model_ptr, efS, topk)
        idx = np.zeros((Q.shape[0], topk), np.uint32)
        dist = np.zeros((Q.shape[0], topk), np.float32)
        lib.pb200_hnsw_resident_fetch(c.m.model_ptr, idx.ctypes.data_as(POINTER(c_uint32)), dist.ctypes.data_as(POINTER(c_float)))
        assert np.array_equal(idx, want[0]) and np.array_equal(dist.view(np.uint32), want[1].view(np.uint32)), (efS, topk)


def test_recorded_reference_outputs(gpu_clib):
    """tests/golden/hnsw_nonfinite (make_golden_hnsw_nonfinite.py): reference-built indices with overwritten rows and the
    reference's own search results, so the engine meets the reference's answer also where oracle/_ref is not built."""
    from oracle import restatement
    from pecos_b200.hnsw import HNSW

    E = np.load(os.path.join(GOLD, "expected.npz"))
    index = json.load(open(os.path.join(GOLD, "expected_index.json")))
    models = {}
    for it in index:
        folder = os.path.join(GOLD, it["model"])
        if it["model"] not in models:
            q = os.path.join(folder, "Q.npz")
            Q = smat.load_npz(q).tocsr() if os.path.exists(q) else np.load(os.path.join(folder, "Q.npy"))
            models[it["model"]] = (HNSW.load(folder), restatement.OracleHNSW(folder, isa=0), Q)
        m, o, Q = models[it["model"]]
        gi, gd = m.predict(Q, pred_params=HNSW.PredParams(efS=it["efS"], topk=it["topk"]), ret_csr=False)
        want = (E[it["key"] + "|idx"], E[it["key"] + "|dist"])
        nf.assert_same_nan_hnsw((gi, gd), want, "engine vs recorded reference " + it["key"])
        nf.assert_same_nan_hnsw((gi, gd), o.predict(Q, it["efS"], it["topk"]), "engine vs restatement " + it["key"])
    assert len(models) >= 3


# ---------------------------------------------------------------------------------------------------------- sharding
def _shard_case(tmp_path, world):
    """Dense d = 70 ip rows in `world` shards (GPU builder), the same overwrites in every shard: a NaN row, +BIG rows (-inf
    distances for the overflow query, tied across shards), -BIG rows (+inf, tied) and a row overflowing both ways (NaN)."""
    from oracle import restatement
    from pecos_b200.hnsw_build import build_hnsw_shards

    rng = np.random.default_rng(40 + world)
    d = 70
    X = nf.dense_rows(rng, 300, d)  # <= 1024 // world rows: a search with topk = 1024 // world returns every row of every shard
    folder = str(tmp_path / f"s{world}")
    build_hnsw_shards(X, folder, world, seed=3, M=8, efC=40, metric="ip", device="cuda:0")
    man = json.load(open(os.path.join(folder, "shards.json")))
    sp = nf.spots(d)
    for r in range(world):
        sub = os.path.join(folder, f"shard-{r}")
        o = restatement.OracleHNSW(sub)
        nan_node = o.init_node if world == 1 else 5  # world 1: the entry node, so every walk is a whole-graph walk
        edits = {nan_node: {sp[1]: np.float32(np.nan)}, 10: {sp[0]: nf.BIG}, 11: {sp[2]: nf.BIG},
                 20: {sp[0]: -nf.BIG}, 21: {sp[-1]: -nf.BIG}, 30: {sp[0]: nf.BIG, sp[-2]: -nf.BIG}}  # (un-fused)
        nf.overwrite_values(sub, edits)
    Q, _ = nf.dense_queries(rng, d, nq=6)
    return folder, man, Q


@pytest.mark.parametrize("world", [2, 3])
def test_sharded_merge_puts_nan_last(tmp_path, gpu_clib, world):
    from .test_hnsw_shard_gpu import _bits_equal, _sharded_predict

    folder, man, Q = _shard_case(tmp_path, world)
    for efS, topk in ((40, 10), (600, 100), (5, 40)):
        (ids, dist), want, _ = _sharded_predict(folder, Q, efS, topk)
        _bits_equal((ids, dist), want, f"world={world} efS={efS} topk={topk}")
        for q in range(Q.shape[0]):
            fin = ~np.isnan(dist[q])
            n = int(fin.sum())
            assert fin[:n].all(), f"a NaN before a number: {dist[q]}"
    # the overflow query with topk >= all rows (every node of every shard returned): -inf at every shard's +BIG rows and
    # +inf at its -BIG rows, tied across shards and taken in rank order, then the NaNs
    topk = 1024 // world
    (ids, dist), want, _ = _sharded_predict(folder, Q, 600, topk)
    _bits_equal((ids, dist), want, f"world={world} efS=600 topk={topk}")
    q = 6
    rb = np.asarray(man["row_begin"])
    for tied in (ids[q][dist[q] == -np.inf], ids[q][dist[q] == np.inf]):
        rank = np.searchsorted(rb, tied, side="right") - 1
        assert tied.size == 2 * world and np.all(np.diff(rank) >= 0), tied
    last = int(np.flatnonzero(dist[q] == np.inf).max())
    assert np.isnan(dist[q][last + 1:last + 1 + 2 * world]).all() and not np.isnan(dist[q][:last]).any()


def test_world1_is_the_unsharded_search_reordered_by_distance_with_nan_last(tmp_path, gpu_clib):
    """A NaN in the reference's heaps can leave its result out of order, NaN and numbers alike (sort_heap under a comparison
    NaN breaks): at world 1 the merge returns the unsharded search's entries ordered by (distance with NaN last, position)."""
    from pecos_b200.distributed import ShardedHNSW
    from pecos_b200.hnsw import HNSW

    from .hnsw_shard_util import hnsw_result_counts
    from .test_hnsw_shard_gpu import _StackComm, _bits_equal

    folder, _, Q = _shard_case(tmp_path, 1)
    s = ShardedHNSW.load(folder, comm=_StackComm(0, 1))
    h = HNSW.load(os.path.join(folder, "shard-0"))
    moved = 0
    for efS, topk in ((40, 10), (600, 100), (5, 40), (10, 10)):
        pp = HNSW.PredParams(efS=efS, topk=topk)
        hi, hd = h.predict(Q, pp, ret_csr=False)
        wi, wd = hi.copy(), hd.copy()
        cnt = hnsw_result_counts(hi, hd)
        for q in range(Q.shape[0]):
            n = int(cnt[q])
            nan = np.isnan(hd[q, :n])
            order = np.lexsort((np.arange(n), np.where(nan, 0, hd[q, :n]), nan))  # (NaN last, distance, position)
            moved += int(not np.array_equal(order, np.arange(n)))
            wi[q, :n], wd[q, :n] = hi[q, order], hd[q, order]
        _bits_equal(s.predict(Q, pp, ret_csr=False), (wi, wd), f"world 1 efS={efS} topk={topk}")
    assert moved > 0  # the overflow and NaN queries: the NaN entry node leaves the heap's output out of order
