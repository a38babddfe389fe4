"""GPU parity tests of HNSW search at the edges of its launch parameters: neighbour lists longer than one warp (maxM0 up to 128,
upper levels with more than 32 neighbours), vector widths from 1 to 12,288 (tail-only rows, 1- and 2-warp CTAs, and widths
whose bulk-copy ring does not fit a warp's shared memory, where the engine runs a shallower ring), indices of 1, 2 and 33
nodes with topk > N and efS < topk, the result heap's move from shared to global memory between ef = 512 and 513 on one
handle, and the sparse query row staging limits.

Every case searches one saved index three ways: the CUDA engine, the C restatement (oracle/restatement.py) -- equal ids and
distance BITS, no tolerance -- and, where oracle/_ref is built, the reference library (bits when it runs the avx512f clone the
kernel restates, or for sparse indices; else ids > 99 % and 1e-5 relative).  Indices are trained by the reference where it
is built, else by this library's builder (util.save_hnsw_index).  Every query batch also holds a copy of a base row, an
all-zero row (every ip distance is exactly 1.0, so the restated heap tie-breaking decides) and one row twice.
"""
from ctypes import c_uint64

import numpy as np
import pytest
import scipy.sparse as smat

from .test_hnsw_build_sparse_cpu import make_rows
from .util import save_hnsw_index

pytestmark = pytest.mark.gpu

GRID = [(10, 10), (64, 10), (200, 10), (5, 40), (600, 100)]
SMEM_WARP_MAX = 200 * 1024   # per-warp shared-memory slice the engine allows (hnsw_engine.cu, ensure_scratch_)
EF_SMEM_MAX = 512            # result heaps up to this many entries live in shared memory


def _unit(rng, n, d):
    X = rng.standard_normal((n, d)).astype(np.float32)
    X /= np.linalg.norm(X, axis=1, keepdims=True)
    return X


def _with_special_rows(Q, X):
    """Q + [a copy of a base row, an all-zero row, Q's second row again]."""
    if smat.issparse(Q):
        out = smat.vstack([Q, X[X.shape[0] // 2], smat.csr_matrix((1, X.shape[1]), dtype=np.float32), Q[1]]).tocsr()
        out = smat.csr_matrix(out, dtype=np.float32)
        out.sort_indices()
        return out
    return np.ascontiguousarray(np.vstack([Q, X[X.shape[0] // 2], np.zeros((1, X.shape[1])), Q[1]]), dtype=np.float32)


def _launch_info(m):
    from pecos_b200.core import get_clib

    out = (c_uint64 * 5)()
    get_clib().clib_float32.pb200_hnsw_launch_info(m.model_ptr, out)
    return dict(zip(("stages", "warps", "ctas", "smem", "heap"), (int(v) for v in out)))


def _expected_slice(d, M, ef, stages):
    """(ring depth, per-warp bytes) the engine must launch: the deepest of `stages`, 4, 0 whose per-warp slice
    [query | ring rows | mbarriers | neighbour ids | distances | result heap if ef <= 512] fits SMEM_WARP_MAX."""
    len16 = d // 16
    vstride = 64 * ((len16 + 3) // 4) + (16 if d % 16 else 0)
    nbmax = (max(2 * M, M) + 31) // 32 * 32
    heap = (ef + 1) * 8 if ef <= EF_SMEM_MAX else 0
    for s in (8, 4, 0):
        if s <= stages:
            per_warp = (vstride * 4 * (1 + s) + 8 * s + nbmax * 8 + heap + 15) & ~15
            if per_warp <= SMEM_WARP_MAX:
                return s, per_warp
    return None, None


class _Index(object):
    """One saved index, searched by the engine, the restatement and (where trained by it) the reference library."""

    def __init__(self, folder, X, M, metric, have_ref, efC=60):
        from oracle import restatement
        from pecos_b200.hnsw import HNSW

        self.sparse = smat.issparse(X)
        self.r = save_hnsw_index(folder, X, M, efC, metric, have_ref)
        self.m = HNSW.load(folder)
        self.o = restatement.OracleHNSW(folder, isa=0)  # avx512f order == what the kernel restates
        self.isa = restatement.host_isa()
        self.want = {}

    def search(self, Q, efS, topk):
        from pecos_b200.hnsw import HNSW

        return self.m.predict(Q, pred_params=HNSW.PredParams(efS=efS, topk=topk), ret_csr=False)

    def check(self, Q, efS, topk, what=""):
        """Engine == restatement (ids, distance bits); the restatement's and the reference's answers are computed once per
        (batch, efS, topk) and reused, e.g. across ring depths."""
        key = (id(Q), efS, topk)
        if key not in self.want:
            oi, od = self.o.predict(Q, efS, topk)
            if self.r is not None:
                ri, rd = self.r.predict(Q, efS, topk, threads=8)
                if self.sparse or self.isa == 0:
                    assert np.array_equal(oi, ri) and np.array_equal(od.view(np.uint32), rd.view(np.uint32)), \
                        f"restatement vs reference library {what} efS={efS} topk={topk}"
                else:  # the reference ran another SIMD clone: summation order differs in the last bits
                    assert np.mean(oi == ri) > 0.99 and np.allclose(od, rd, rtol=1e-5, atol=1e-6), \
                        f"restatement vs reference library {what} efS={efS} topk={topk}"
            self.want[key] = (oi, od)
        oi, od = self.want[key]
        idx, dist = self.search(Q, efS, topk)
        assert np.array_equal(idx, oi), f"ids vs restatement {what} efS={efS} topk={topk}"
        assert np.array_equal(dist.view(np.uint32), od.view(np.uint32)), f"distance bits vs restatement {what} efS={efS} topk={topk}"
        return idx, dist


@pytest.mark.parametrize("d", [64, 128])
@pytest.mark.parametrize("metric", ["ip", "l2"])
@pytest.mark.parametrize("M", [17, 32, 48, 64])
def test_dense_neighbour_lists_past_one_warp(tmp_path, gpu_clib, have_ref, M, metric, d):
    """maxM0 = 2M in {34, 64, 96, 128}: two to four 32-lane rounds of the visited test-and-set and compaction per expansion,
    nb_ids scratch past 32 slots; M >= 33 also walks more than 32 neighbours per upper-level hop."""
    rng = np.random.default_rng(1000 * M + d + (metric == "l2"))
    X = _unit(rng, 3000, d)
    ix = _Index(str(tmp_path / "idx"), X, M, metric, have_ref)
    assert ix.o.maxM0 == 2 * M and ix.o.l0_max_degree == 2 * M
    Q = _with_special_rows(_unit(rng, 100, d), X)
    for efS, topk in GRID:
        ix.check(Q, efS, topk, f"M={M}")


@pytest.mark.parametrize("M,metric", [(32, "ip"), (48, "l2")])
def test_sparse_neighbour_lists_past_one_warp(tmp_path, gpu_clib, have_ref, M, metric):
    X = make_rows(M, 3000, 20000, 60, 61)
    ix = _Index(str(tmp_path / "idx"), X, M, metric, have_ref)
    Q = _with_special_rows(make_rows(M + 1, 100, 20000, 60, 0), X)
    for efS, topk in GRID:
        ix.check(Q, efS, topk, f"csr M={M}")


# (d, metric): tail-only rows, an exact 16-wide block, block + tail, a 64-wide chunk +- 1; then 2- and 1-warp CTAs; then widths
# whose 4- or 8-deep ring does not fit one warp's slice (6,144 and 8,192 at depth 8; 10,129 / 10,176 at the edge of depth 4,
# where the result heap in shared memory decides; 12,288 at every depth but 0)
DIMS = [(1, "ip"), (4, "l2"), (15, "ip"), (16, "l2"), (17, "ip"), (63, "l2"), (65, "ip"),
        (1024, "l2"), (1536, "ip"), (3072, "l2"), (4096, "ip"), (6144, "l2"), (8192, "ip"),
        (10129, "l2"), (10176, "ip"), (12288, "l2")]
DIM_M = 16


@pytest.mark.parametrize("d,metric", DIMS)
def test_dense_dimensions_and_ring_depth_fallback(tmp_path, gpu_clib, have_ref, d, metric):
    """Every ring depth setting (0, 4, 8) gives the restatement's bits; the engine runs the deepest depth up to the setting
    whose per-warp slice fits, with the launch geometry that follows from it."""
    rng = np.random.default_rng(d)
    wide = d >= 1024
    X = _unit(rng, 1500 if wide else 2000, d)
    ix = _Index(str(tmp_path / "idx"), X, DIM_M, metric, have_ref)
    Q = _with_special_rows(_unit(rng, 32 if wide else 100, d), X)
    grid = [(100, 10), (512, 10), (513, 10)] if d > 10000 else [(64, 10), (600, 20)]
    c = gpu_clib.clib_float32
    for stages in (0, 4, 8):
        assert c.pb200_hnsw_set_stages(ix.m.model_ptr, stages) == stages
        for efS, topk in grid:
            ix.check(Q, efS, topk, f"d={d} stages={stages}")
            depth, per_warp = _expected_slice(d, DIM_M, max(efS, topk), stages)
            info = _launch_info(ix.m)
            assert info["stages"] == depth and info["smem"] == info["warps"] * per_warp, (d, stages, efS, info)
            assert info["warps"] >= 1 and info["warps"] * per_warp <= max(96 * 1024, per_warp)
    # the depths the wide rows must fall back to (from the slice sizes above, not from the engine)
    if d == 12288:
        assert _expected_slice(d, DIM_M, 100, 8)[0] == 0
    if d == 10176:
        assert [_expected_slice(d, DIM_M, ef, 4)[0] for ef in (100, 512, 513)] == [4, 0, 4]
    if d == 10129:
        assert _expected_slice(d, DIM_M, 100, 4)[0] == 0
    if d in (6144, 8192):
        assert _expected_slice(d, DIM_M, 64, 8)[0] == 4


@pytest.mark.parametrize("N", [1, 2, 33])
@pytest.mark.parametrize("metric", ["ip", "l2"])
def test_tiny_indices_and_result_trimming(tmp_path, gpu_clib, have_ref, N, metric):
    """topk > N (the tail stays zeros, as c_ann_hnsw_predict_* leaves it), efS < topk, efS = 0 with topk > 0."""
    rng = np.random.default_rng(N + 50)
    X = _unit(rng, N, 24)
    ix = _Index(str(tmp_path / "idx"), X, 8, metric, have_ref)
    Q = _with_special_rows(_unit(rng, 40, 24), X)
    for efS, topk in [(10, 10), (3, 10), (0, 5), (0, 40), (1, 1), (50, 40), (200, 3)]:
        idx, dist = ix.check(Q, efS, topk, f"N={N}")
        assert not idx[:, N:].any() and not dist[:, N:].view(np.uint32).any()


def test_result_heap_placement_and_scratch_reuse(tmp_path, gpu_clib, have_ref):
    """One handle, ef up and down across the shared / global result-heap switch: every call equals the restatement, the
    global heap grows with ef, is kept when ef shrinks, and the slice shrinks by the heap once ef > 512."""
    rng = np.random.default_rng(128)
    X = _unit(rng, 3000, 128)
    ix = _Index(str(tmp_path / "idx"), X, 32, "ip", have_ref)
    Q = _with_special_rows(_unit(rng, 200, 128), X)
    info = {}
    for efS in (512, 513, 600, 1000, 100, 700, 10):
        ix.check(Q, efS, 10)
        info[efS] = _launch_info(ix.m)
        depth, per_warp = _expected_slice(128, 32, efS, 4)
        assert info[efS]["stages"] == depth == 4 and info[efS]["smem"] == info[efS]["warps"] * per_warp, (efS, info[efS])
    assert info[512]["heap"] == 0
    # the per-warp slice holds the heap (513 entries of 8 bytes) at ef = 512 and not at ef = 513
    assert info[512]["warps"] == info[513]["warps"]
    assert info[512]["smem"] - info[513]["smem"] >= info[512]["warps"] * 513 * 8
    assert info[600]["smem"] == info[700]["smem"] == info[1000]["smem"] == info[513]["smem"]
    # global heap: (warps in the grid) x (ef + 1) entries, grown for 513 -> 600 -> 1000, then reused
    h513, h600, h1000 = info[513]["heap"], info[600]["heap"], info[1000]["heap"]
    assert h513 > 0 and h513 % 514 == 0 and h600 % 601 == 0 and h1000 % 1001 == 0
    assert h513 // 514 == h600 // 601 == h1000 // 1001
    assert info[100]["heap"] == info[700]["heap"] == info[10]["heap"] == h1000


def test_sparse_query_staging_limits(tmp_path, gpu_clib, have_ref):
    """Query rows of exactly 4,096 entries (staged in shared memory) and 4,097 (searched in global memory), and one of 20,000
    entries that sets every bit of the 8,192-bit membership filter, in one batch."""
    D = 30000
    X = make_rows(7, 2000, D, 80, 61)
    ix = _Index(str(tmp_path / "idx"), X, 16, "ip", have_ref)
    rng = np.random.default_rng(9)
    rows = []
    for k in (4096, 4097, 20000):
        c = np.arange(k) if k == 20000 else np.sort(rng.choice(D, size=k, replace=False))
        v = np.abs(rng.standard_normal(k)).astype(np.float32) + np.float32(0.01)
        rows.append(smat.csr_matrix((v / np.linalg.norm(v), c, [0, k]), shape=(1, D), dtype=np.float32))
    h = ((np.arange(20000, dtype=np.uint64) * np.uint64(2654435761)) & np.uint64(0xFFFFFFFF)) >> np.uint64(19)
    assert np.unique(h).size == 8192  # the filter hash of csrc/hnsw_engine.cu (sp_hash): every bit set
    Q = _with_special_rows(smat.vstack([make_rows(8, 30, D, 80, 0)] + rows).tocsr(), X)
    assert sorted(np.diff(Q.indptr))[-3:] == [4096, 4097, 20000]
    for efS, topk in [(64, 10), (600, 100)]:
        ix.check(Q, efS, topk, "csr staging")


# (M, widest d that fits, first d that does not): for a width that is not a multiple of 16 and for one that is.  The limit is
# 4 * dense_vstride(d) + 8 * nbmax <= 204,800 bytes (depth 0, the result heap in global memory), whatever ef.
WIDEST = [(16, 51087, 51089), (16, 51136, 51152), (48, 50959, 50961), (48, 51008, 51024)]


@pytest.mark.parametrize("M,d_fit,d_over", WIDEST)
def test_widest_dense_rows_search_and_one_more_raises(tmp_path, gpu_clib, have_ref, M, d_fit, d_over):
    """The widest rows run depth 0 with the result heap in global memory where the slice needs it (every ef), equal to the
    restatement; one more 16-block makes predict raise ValueError before any native call, and the process lives on."""
    from pecos_b200.hnsw import HNSW

    from .test_hnsw_nonfinite_cpu import dense_plan_rule

    rng = np.random.default_rng(d_fit)
    X = _unit(rng, 40, d_fit)
    ix = _Index(str(tmp_path / "fit"), X, M, "ip", have_ref, efC=20)
    Q = _with_special_rows(_unit(rng, 5, d_fit), X)
    for efS, topk in [(10, 10), (100, 10), (512, 10), (513, 10)]:
        ix.check(Q, efS, topk, f"d={d_fit} M={M}")
        fits, plan = gpu_clib.hnsw_search_fits(ix.m.model_ptr, efS, topk)
        want = dense_plan_rule(d_fit, 2 * M, 4, max(efS, topk))
        assert fits and want[0] and (plan["stages"], bool(plan["heap_in_smem"]), plan["per_warp_bytes"]) == want[1:]
        info = _launch_info(ix.m)
        assert info["stages"] == 0 and info["smem"] == info["warps"] * plan["per_warp_bytes"], (efS, info, plan)
        assert plan["heap_in_smem"] or info["heap"] >= max(efS, topk) + 1
    assert not gpu_clib.hnsw_search_fits(ix.m.model_ptr, 512, 10)[1]["heap_in_smem"]
    Xo = _unit(rng, 40, d_over)
    save_hnsw_index(str(tmp_path / "over"), Xo, M, 20, "ip", have_ref)
    wide = HNSW.load(str(tmp_path / "over"))  # loading and creating searchers stay allowed, as in the reference
    wide.searchers_create(2)
    launches = (c_uint64 * 8)()
    gpu_clib.clib_float32.pb200_hnsw_get_info(wide.model_ptr, launches)
    before = int(launches[7])
    for efS in (10, 512, 513):
        assert not gpu_clib.hnsw_search_fits(wide.model_ptr, efS, 10)[0]
        with pytest.raises(ValueError, match="cannot be searched"):
            wide.predict(_unit(rng, 3, d_over), pred_params=HNSW.PredParams(efS=efS, topk=10), ret_csr=False)
    gpu_clib.clib_float32.pb200_hnsw_get_info(wide.model_ptr, launches)
    assert int(launches[7]) == before
    ix.check(Q, 64, 10, "after the refusal")


def test_heap_leaves_shared_memory_below_ef_513(tmp_path, gpu_clib, have_ref):
    """d = 50,500 with M = 16 fits depth 0 with the heap in shared memory at ef = 100 but not at ef = 512: the heap moves to
    global memory there, on one handle, between calls."""
    rng = np.random.default_rng(50500)
    X = _unit(rng, 40, 50500)
    ix = _Index(str(tmp_path / "i"), X, 16, "l2", have_ref, efC=20)
    Q = _with_special_rows(_unit(rng, 5, 50500), X)
    placed = {}
    for efS in (100, 512, 100, 600):
        ix.check(Q, efS, 10, f"ef={efS}")
        fits, plan = gpu_clib.hnsw_search_fits(ix.m.model_ptr, efS, 10)
        info = _launch_info(ix.m)
        assert fits and info["stages"] == 0 and info["smem"] == info["warps"] * plan["per_warp_bytes"]
        placed[efS] = plan["heap_in_smem"]
    assert placed == {100: 1, 512: 0, 600: 0}
