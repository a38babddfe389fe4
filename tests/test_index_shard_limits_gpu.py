"""GPU tests of index sharding at the limits of its kernels.

Index sharding splits XR-Linear's leaf layer over ranks (the chunks a rank does not own are flagged absent, kChunkAbsent)
or keeps one HNSW graph per shard; every rank packs its local top-k into 16-byte {key, id, value} records, ONE all-gather
stacks them as [world][rows][stride], and shard_merge_packed_kernel (csrc/shard_merge.cuh) keeps the k largest keys per
query.  Here several shard handles on one GPU emulate the ranks and a stacking comm emulates the all-gather (two passes: each
rank's own records first, then the merge of all of them).

* The merge kernel against numpy on hand-built records, at its capacity of world x stride = 1024 keys per query and off
  powers of two, with row counts that are not a multiple of its 4 warps per CTA.
* XR-Linear through ShardedXLinearModel in every kernel mode (pb200_xlinear_set_lookup 0 - 7, set on every shard handle):
  the merged result is bit-identical to the unsharded prediction in the same mode, which matches the C restatement and the
  float64 path scores; each rank's sent records equal its expected local list (the unsharded full candidate order kept to
  the rank's leaf chunks); keys are non-zero exactly below the count, strictly decreasing, carry the orderable score with
  +-0 folded in the high word and distinct candidate positions across ranks.  The kernels seen on ranks with absent chunks
  are collected and the last test asserts that every leaf score kernel of the csr path, the prefix launch, and every top-k
  kernel and branch a sharded call can take ran there.  The block top-k's HBM-sort branch needs k > 1,024, which no
  sharded call can have (world >= 2 and world x stride <= 1024), so it is not part of that list.
* Shard-split edges (more ranks than leaf chunks, one chunk holding most bytes, a permuted leaf), a tiled call, and the
  merge capacity of both engines: 1024 records per query pass, more raise ValueError before any GPU work.

Score kernel ids: 0 row lists, 1 feature map, 2 dense (not on the csr-only sharded path), 3 query-warp, 4 chunk-major.
Top-k ids: 0 block sort, 1 warp select, 2 estimate filter.
"""
import os
from ctypes import POINTER, c_double, c_float, c_int, c_uint32, c_uint64

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .hnsw_shard_util import hnsw_rows
# _hnsw_sharded_predict: every rank's ShardedHNSW.predict against merge_hnsw_shards_numpy of the per-shard searches
from .test_hnsw_shard_gpu import _bits_equal, _records, _sharded_predict as _hnsw_sharded_predict, _StackComm
from .test_xlinear_limits_gpu import _f64_check, _queries, _same_bits, _two_layer
from .util import assert_csr_parity, random_tree

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CAP = 1024       # merge capacity: world x stride records per query (kSelKeys)
SORT_CAP = 2048  # block top-k: one sort up to this many candidates per query, streaming beyond (kSortCap)
MODES = list(range(8))
PPS = ("l3-hinge", "noop", "sigmoid", "log-l2-hinge")

# (leaf score kernel | "prefix" | top-k kernel and branch) seen on a rank that has absent leaf chunks
_SEEN = set()


# ------------------------------------------------------------------------------------------------ merge kernel vs numpy
def _pack(keys, ids, vals):
    """[world][rows][stride] keys u64, ids u32, values f32 -> the records as int64 pairs (torch's view of the exchange)."""
    hi = np.asarray(vals, dtype=np.float32).view(np.uint32).astype(np.uint64) << np.uint64(32)
    return np.stack([keys.view(np.int64), (ids.astype(np.uint64) | hi).view(np.int64)], axis=-1)


def _hand_records(seed, world, rows, stride, n_ids):
    """Records whose rows cycle through: all empty; a few records (fewer than any k); one rank holding every record; equal
    high words (the low word decides); high words from negative and positive scores (bit 31 clear and set); the largest
    and smallest non-zero keys among full rows.  Keys are unique per row (distinct low words)."""
    rng = np.random.default_rng(seed)
    n = world * stride
    # distinct low words per row: (a + i * b) mod 2^31 with b odd, plus 2, shuffled; never 0, 1 or 0xFFFFFFFF
    a = rng.integers(0, 1 << 31, size=(rows, 1), dtype=np.uint64)
    b = rng.integers(0, 1 << 30, size=(rows, 1), dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    low = (a + np.arange(n, dtype=np.uint64)[None, :] * b) % np.uint64(1 << 31) + np.uint64(2)
    low = np.take_along_axis(low, np.argsort(rng.random((rows, n)), axis=1), axis=1)
    high = rng.integers(0, 1 << 32, size=(rows, n), dtype=np.uint64)
    valid = np.ones((rows, n), dtype=bool)
    kind = (np.arange(rows) + seed) % 6
    valid[kind == 0] = False
    valid[kind == 1] = rng.random((int((kind == 1).sum()), n)) < min(0.1, 3.0 / n) + 1e-9
    owner = (np.arange(n) // stride)[None, :]
    valid[kind == 2] = (owner == (np.arange(rows)[kind == 2] % world)[:, None])
    high[kind == 3] = np.uint64(0xBF800000)  # one high word for the whole row
    s = rng.standard_normal((rows, n)).astype(np.float32)
    u = s.view(np.uint32).astype(np.uint64)
    orderable = np.where(u & np.uint64(0x80000000), ~u & np.uint64(0xFFFFFFFF), u | np.uint64(0x80000000))
    high[kind == 4] = orderable[kind == 4]
    keys = (high << np.uint64(32)) | low
    for r in np.nonzero(kind == 5)[0]:  # n >= 5 in every shape here
        i, j = rng.choice(n, size=2, replace=False)
        keys[r, i] = np.uint64(0xFFFFFFFFFFFFFFFF)
        keys[r, j] = np.uint64(1)
    keys = np.where(valid, keys, np.uint64(0))
    ids = np.where(valid, rng.integers(0, n_ids, size=(rows, n)), 0).astype(np.uint32)
    vals = np.where(valid, rng.standard_normal((rows, n)), 0).astype(np.float32)
    vals[valid & (rng.random((rows, n)) < 0.05)] = np.float32(-0.0)
    shape = (rows, world, stride)
    to_wrs = lambda x: np.ascontiguousarray(x.reshape(shape).transpose(1, 0, 2))  # noqa: E731
    return to_wrs(keys), to_wrs(ids), to_wrs(vals)


def _numpy_merge(keys, ids, vals, k):
    """Top-min(k, non-zero keys) records per query by unsigned key: (ids, value bits, counts), rows x k with zero tails."""
    world, rows, stride = keys.shape
    K = np.ascontiguousarray(keys.transpose(1, 0, 2)).reshape(rows, -1)
    I = np.ascontiguousarray(ids.transpose(1, 0, 2)).reshape(rows, -1)
    V = np.ascontiguousarray(vals.transpose(1, 0, 2)).reshape(rows, -1).view(np.uint32)
    order = np.argsort(K, axis=1, kind="stable")[:, ::-1][:, :k]
    cnt = np.minimum((K != 0).sum(1), k)
    live = np.arange(order.shape[1])[None, :] < cnt[:, None]
    out_i = np.zeros((rows, k), dtype=np.uint32)
    out_v = np.zeros((rows, k), dtype=np.uint32)
    out_i[:, :order.shape[1]] = np.where(live, np.take_along_axis(I, order, 1), 0)
    out_v[:, :order.shape[1]] = np.where(live, np.take_along_axis(V, order, 1), 0)
    return out_i, out_v, cnt


@pytest.fixture(scope="module")
def merge_handles(tmp_path_factory, gpu_clib):
    """An XR-Linear model of 640 labels and a small HNSW index: the merge entry points of both engines."""
    from pecos_b200.hnsw import HNSW
    from pecos_b200.xlinear import XLinearModel

    folder = str(tmp_path_factory.mktemp("merge") / "m")
    synth.save_xlinear_model(folder, random_tree(801, [4, 32, 640], 100, 8, bias=1.0), bias=1.0, only_topk=10)
    xl = XLinearModel.load(folder, is_predict_only=True)
    hn = HNSW.load(os.path.join(ROOT, "tests", "golden", "hnsw_toy", "model_l2"))
    return xl, hn, 640


@pytest.mark.parametrize("world,stride", [(1, 1024), (2, 512), (8, 128), (3, 341), (5, 1), (1, 5)])
@pytest.mark.parametrize("rows", [1, 3, 4, 5, 4097])
def test_merge_kernel_equals_numpy(merge_handles, gpu_clib, world, stride, rows):
    import torch

    from pecos_b200.core import ScipyCompressedSparseAllocator

    xl, hn, n_ids = merge_handles
    c = gpu_clib.clib_float32
    keys, ids, vals = _hand_records(world * 1000 + stride * 7 + rows, world, rows, stride, n_ids)
    g = torch.from_numpy(_pack(keys, ids, vals)).cuda().contiguous()
    torch.cuda.synchronize()
    n = world * stride
    for k in sorted({1, stride, n, n + 7}):
        k_out = min(k, n)
        want_i, want_v, want_c = _numpy_merge(keys, ids, vals, k_out)
        alloc = ScipyCompressedSparseAllocator()
        c.pb200_xlinear_sharded_merge_packed(xl.model.model_chain, world, rows, stride, k, g.data_ptr(), alloc.cfunc)
        what = f"xlinear merge world={world} stride={stride} rows={rows} k={k}"
        assert alloc.rows == rows and alloc.cols == n_ids, what
        assert np.array_equal(np.diff(alloc.indptr.astype(np.int64)), want_c), f"{what}: row counts"
        live = np.arange(k_out)[None, :] < want_c[:, None]
        assert np.array_equal(alloc.indices, want_i[live]), f"{what}: ids"
        assert np.array_equal(alloc.data.view(np.uint32), want_v[live]), f"{what}: value bits"
    # HNSW: stride = topk, rows x topk arrays with zero tails
    want_i, want_v, _ = _numpy_merge(keys, ids, vals, stride)
    got_i = np.full((rows, stride), 7, dtype=np.uint32)
    got_v = np.full((rows, stride), 7.0, dtype=np.float32)
    c.pb200_hnsw_sharded_merge_packed(hn.model_ptr, world, rows, stride, g.data_ptr(), got_i.ctypes.data_as(POINTER(c_uint32)),
                                      got_v.ctypes.data_as(POINTER(c_float)))
    what = f"hnsw merge world={world} stride={stride} rows={rows}"
    assert np.array_equal(got_i, want_i), f"{what}: ids"
    assert np.array_equal(got_v.view(np.uint32), want_v), f"{what}: value bits"


# ------------------------------------------------------------------------------------------------ XR-Linear sharded runs
def _orderable_folded(bits):
    """High word of an XR-Linear key: orderable(score) with -0.0 folded onto +0.0."""
    u = np.where((bits & np.uint32(0x7FFFFFFF)) == 0, np.uint32(0), bits).astype(np.uint64)
    return np.where(u & np.uint64(0x80000000), ~u & np.uint64(0xFFFFFFFF), u | np.uint64(0x80000000))


class _Case(object):
    """One model: the unsharded predict-only handle, its layers and the owner chunk of every leaf label, and the shard
    handles of every world asked for (loaded through ShardedXLinearModel.load with stacking comms)."""

    def __init__(self, gpu_clib, folder, layers):
        from pecos_b200.xlinear import XLinearModel

        self.clib, self.c = gpu_clib, gpu_clib.clib_float32
        self.folder, self.layers, self.depth = folder, layers, len(layers)
        self.whole = XLinearModel.load(folder, is_predict_only=True)
        self.h = self.whole.model.model_chain
        C = smat.csr_matrix(layers[-1][1])
        assert np.all(np.diff(C.indptr) == 1)
        self.chunk_of = C.indices.astype(np.int64)  # leaf chunk p holds the children of node p of the layer above
        self.n_chunks = C.shape[1]
        self._shards = {}

    def shards(self, world):
        from pecos_b200.distributed import ShardedXLinearModel

        if world not in self._shards:
            ms = [ShardedXLinearModel.load(self.folder, comm=_StackComm(r, world)) for r in range(world)]
            for r, m in enumerate(ms):
                assert m.shard[:2] == (r, world)
            assert ms[0].shard[2] == 0 and ms[-1].shard[3] == self.n_chunks
            assert all(ms[r].shard[3] == ms[r + 1].shard[2] for r in range(world - 1))
            self._shards[world] = ms
        return self._shards[world]

    def ids(self, h):
        kid = (c_int * (2 * self.depth))()
        self.c.pb200_xlinear_get_kernel_ids(h, kid)
        return [(kid[2 * d], kid[2 * d + 1]) for d in range(self.depth)]

    def prefix_used(self, h):
        prof = (c_double * (2 * self.depth))()
        self.c.pb200_xlinear_get_profile(h, prof)
        return self.depth >= 2 and prof[1] == 0.0 and prof[2] == 0.0

    def unsharded(self, X, beam, topk, pp, mode):
        self.c.pb200_xlinear_set_lookup(self.h, mode)
        try:
            return self.whole.predict(X, beam_size=beam, only_topk=topk, post_processor=pp)
        finally:
            self.c.pb200_xlinear_set_lookup(self.h, 1)

    def reference(self, X, beam, topk, pp):
        """Mode 1's unsharded result checked against the restatement and the float64 path scores, and every candidate of
        the leaf in rank order (only_topk = the leaf's candidate-row width), checked against the restatement's order."""
        from oracle.restatement import OracleXLinear

        want = self.unsharded(X, beam, topk, pp, 1)
        o = OracleXLinear(os.path.join(self.folder, "ranker"))
        what = f"{os.path.basename(self.folder)} beam={beam} topk={topk} {pp}"
        assert_csr_parity(want, o.predict(X, beam, pp, topk), what=f"{what} vs the restatement")
        _f64_check(self.layers, 1.0, X, want, pp, what=what)
        width = self.clib.xlinear_plan_stride(self.h, beam, 1 << 30)  # beam entering the leaf x its widest chunk
        full = self.unsharded(X, beam, width, pp, 1)
        ref_full = o.predict(X, beam, pp, 10_000)
        assert np.array_equal(full.indptr, ref_full.indptr) and np.array_equal(full.indices, ref_full.indices), (
            f"{what}: full candidate order differs from the restatement")
        return want, full

    def local_lists(self, full, world, stride):
        """Per rank: (ids, value bits, count) rows x stride, the first `stride` candidates of the full order whose leaf
        chunk lies in the rank's range."""
        rows = full.shape[0]
        n = np.diff(full.indptr)
        W = max(int(n.max(initial=0)), 1)
        lab = np.full((rows, W), -1, dtype=np.int64)
        bits = np.zeros((rows, W), dtype=np.uint32)
        live = np.arange(W)[None, :] < n[:, None]
        lab[live] = full.indices
        bits[live] = np.asarray(full.data, dtype=np.float32).view(np.uint32)
        chunk = np.where(live, self.chunk_of[np.maximum(lab, 0)], -1)
        out = []
        for m in self.shards(world):
            c0, c1 = m.shard[2:]
            own = live & (chunk >= c0) & (chunk < c1)
            order = np.argsort(~own, axis=1, kind="stable")[:, :stride]
            cnt = np.minimum(own.sum(1), stride)
            keep = np.arange(order.shape[1])[None, :] < cnt[:, None]
            ids = np.zeros((rows, stride), dtype=np.uint32)
            vb = np.zeros((rows, stride), dtype=np.uint32)
            ids[:, :order.shape[1]] = np.where(keep, np.take_along_axis(lab, order, 1), 0)
            vb[:, :order.shape[1]] = np.where(keep, np.take_along_axis(bits, order, 1), 0)
            out.append((ids, vb, cnt))
        return out

    def sharded(self, X, world, beam, topk, pp, mode):
        """Every rank's ShardedXLinearModel.predict with the all-gather emulated: pass 1 sends each rank's records, pass 2
        merges them on the first and last rank.  Returns (merged result, sent records per rank, per-rank (leaf kernel ids,
        prefix used, rank has absent chunks))."""
        ms = self.shards(world)
        sent, info = [], []
        for m in ms:
            h = m.model_chain
            self.c.pb200_xlinear_set_lookup(h, mode)
            self.c.pb200_xlinear_set_profile(h, 1)
            self.c.pb200_xlinear_reset_profile(h)
            m.comm.parts = None
            m.predict(X, beam_size=beam, only_topk=topk, post_processor=pp)
            self.c.pb200_xlinear_set_profile(h, 0)
            sent.append(m.comm.sent)
            c0, c1 = m.shard[2:]
            info.append((self.ids(h)[-1], self.prefix_used(h), c1 - c0 < self.n_chunks))
            assert m.last_exchange_bytes == 16 * X.shape[0] * sent[-1].shape[1]
        got = None
        for r in sorted({0, world - 1}):
            ms[r].comm.parts = sent
            res = ms[r].predict(X, beam_size=beam, only_topk=topk, post_processor=pp)
            if got is None:
                got = res
            else:
                _same_bits(res, got, f"rank {r} vs rank 0")
        for m in ms:
            self.c.pb200_xlinear_set_lookup(m.model_chain, 1)
        return got, sent, info


def _check_records(sent, expected, what):
    """Each rank's records equal its expected local list; key rules; distinct candidate positions across ranks."""
    lows = []
    for r, (rec, (w_ids, w_bits, w_cnt)) in enumerate(zip(sent, expected)):
        keys, ids, bits = _records(rec)
        wr = f"{what} rank {r}"
        assert keys.shape == w_ids.shape, f"{wr}: stride {keys.shape[1]}, expected {w_ids.shape[1]}"
        assert np.array_equal(ids, w_ids), f"{wr}: record ids differ from the rank's expected local list"
        assert np.array_equal(bits, w_bits), f"{wr}: record value bits differ from the expected local list"
        slot = np.arange(keys.shape[1])[None, :]
        live = slot < w_cnt[:, None]
        assert np.array_equal(keys != 0, live), f"{wr}: non-zero keys are not exactly the slots below the count"
        dec = (keys[:, 1:] < keys[:, :-1]) | ~live[:, 1:]
        assert dec.all(), f"{wr}: keys not strictly decreasing"
        hi = keys >> np.uint64(32)
        assert np.array_equal(np.where(live, hi, 0), np.where(live, _orderable_folded(bits), 0)), f"{wr}: key high words"
        lows.append(np.where(live, keys & np.uint64(0xFFFFFFFF), 0))
    low = np.sort(np.concatenate(lows, axis=1), axis=1)
    dup = (low[:, 1:] == low[:, :-1]) & (low[:, 1:] != 0)
    assert not dup.any(), f"{what}: candidate positions repeat across ranks"


def _note_coverage(info, topk, cand_counts):
    for (score, topk_id), prefix, absent in info:
        if not absent:
            continue
        _SEEN.add(f"score {score}")
        if prefix:
            _SEEN.add("prefix")
        if topk_id == 0:
            if cand_counts.max() <= SORT_CAP:
                _SEEN.add("block top-k, one sort")
            elif cand_counts.min() > SORT_CAP and topk <= SORT_CAP // 2:
                _SEEN.add("block top-k, streaming")
        elif topk_id == 1:
            _SEEN.add("warp select, k > 32" if topk > 32 else "warp select")
        elif topk_id == 2:
            _SEEN.add("estimate filter")


def _run(case, X, worlds, beam, topk, pps=PPS, modes=MODES):
    """Every check of a sharded XR-Linear call, for each (pp, world, mode) of one (beam, topk) call of `case`; returns the
    unsharded mode-1 result of the last pp."""
    for pp in pps:
        want, full = case.reference(X, beam, topk, pp)
        base = {m: case.unsharded(X, beam, topk, pp, m) for m in modes}
        for m in modes:
            _same_bits(base[m], want, f"unsharded mode {m} vs mode 1, {pp}")
        stride = case.clib.xlinear_plan_stride(case.h, beam, topk)
        cand = np.diff(full.indptr)
        for world in worlds:
            expected = case.local_lists(full, world, stride)
            for mode in modes:
                what = f"{os.path.basename(case.folder)} world={world} beam={beam} topk={topk} {pp} mode {mode}"
                got, sent, info = case.sharded(X, world, beam, topk, pp, mode)
                _same_bits(got, base[mode], what)
                _check_records(sent, expected, what)
                _note_coverage(info, topk, cand)
    return want


def _save(folder, layers, only_topk=10):
    synth.save_xlinear_model(folder, layers, bias=1.0, only_topk=only_topk)
    return folder


@pytest.fixture(scope="module")
def three_layer(tmp_path_factory, gpu_clib):
    """5 / 40 / 640 nodes, contiguous (the prefix launch scores layers 0 and 1 in mode 5 and feeds the sharded leaf)."""
    layers = random_tree(701, [5, 40, 640], 400, 30, bias=1.0)
    return _Case(gpu_clib, _save(str(tmp_path_factory.mktemp("three") / "m"), layers), layers), 400


@pytest.fixture(scope="module")
def permuted(tmp_path_factory, gpu_clib):
    """8 / 64 / 900 nodes with shuffled child -> parent assignments: the leaf is permuted (label_of_col)."""
    layers = random_tree(711, [8, 64, 900], 400, 30, bias=1.0, permute=True)
    return _Case(gpu_clib, _save(str(tmp_path_factory.mktemp("perm") / "m"), layers), layers), 400


@pytest.fixture(scope="module")
def wide_leaf(tmp_path_factory, gpu_clib):
    """Layer 0: one chunk of 48 nodes; leaf: 48 chunks of exactly 64 columns.  Beam 40 puts 2,560 candidates in every
    leaf row (past the block top-k's single sort), beam 2 puts 128."""
    layers = _two_layer(721, [64] * 48, 500, 12)
    return _Case(gpu_clib, _save(str(tmp_path_factory.mktemp("wide") / "m"), layers), layers), 500


@pytest.mark.parametrize("beam,topk", [(6, 10), (6, 48)])
def test_three_layer_model_through_every_leaf_kernel(three_layer, beam, topk):
    """k = 10 takes the estimate filter by default, k = 48 the warp select; modes 0 (row lists + block sort), 2 (feature
    map), 3 (query-warp), 5 (chunk-major + prefix launch) and the rest on a sharded leaf."""
    case, D = three_layer
    X = _queries(702, D, [40] * 200 + [150])
    _run(case, X, (2, 3, 8), beam, topk)


def test_permuted_leaf_every_mode(permuted):
    case, D = permuted
    X = _queries(712, D, [30] * 150 + [120])
    L = case.clib.host_model_layout(os.path.join(case.folder, "ranker"))[-1]
    assert L["label_of_col"].size == L["n_cols"]  # the leaf's columns are stored out of label order
    _run(case, X, (2, 3, 8), 9, 12)


def test_saturated_ties_are_ordered_by_global_position(tmp_path, gpu_clib):
    """Saturated hinge: most scores are exactly 1.0, so only the candidate position in the key orders them, across ranks."""
    layers = random_tree(731, [6, 48, 600], 200, 40, bias=1.0, permute=True, saturate=True)
    case = _Case(gpu_clib, _save(str(tmp_path / "m"), layers), layers)
    X = _queries(732, 200, [50] * 120 + [90])
    want = _run(case, X, (2, 3, 8), 10, 10, pps=("l3-hinge",))
    assert np.mean(want.data == 1.0) > 0.2


def test_streaming_block_topk_at_the_merge_capacity(wide_leaf):
    """World 2, k = 512 over 2,560 candidates per row: the block top-k streams (k <= 1,024), and 2 x 512 = 1,024 records
    per query fill the merge kernel."""
    case, D = wide_leaf
    X = _queries(722, D, [40] * 90 + [120])
    _run(case, X, (2,), 40, 512, pps=("l3-hinge", "log-l2-hinge"))


# ------------------------------------------------------------------------------------------------ shard-split edges
def test_more_ranks_than_leaf_chunks(tmp_path, gpu_clib):
    """6 leaf chunks over 8 ranks: the ranks that own nothing load, and send only empty records in every mode."""
    layers = random_tree(741, [3, 6, 60], 200, 20, bias=1.0)
    case = _Case(gpu_clib, _save(str(tmp_path / "m"), layers), layers)
    assert case.n_chunks == 6
    X = _queries(742, 200, [30] * 60 + [80])
    _run(case, X, (8,), 4, 10, pps=("l3-hinge", "noop"))
    empty = [m for m in case.shards(8) if m.shard[2] == m.shard[3]]
    assert len(empty) >= 2
    for m in empty:
        assert int((m.comm.sent != 0).sum()) == 0


def test_one_chunk_holding_most_bytes_leaves_middle_ranks_empty(tmp_path, gpu_clib):
    """Leaf chunks of 4 columns around one of 200 (about 80% of the entry bytes): the byte-balanced split gives ranks 1 and
    2 of 4 nothing, between two ranks that own chunks."""
    layers = _two_layer(751, [4] * 5 + [200] + [4] * 5, 300, 12)
    case = _Case(gpu_clib, _save(str(tmp_path / "m"), layers), layers)
    X = _queries(752, 300, [30] * 80 + [100])
    ranges = [m.shard[2:] for m in case.shards(4)]
    assert ranges[0][0] < ranges[0][1] and ranges[3][0] < ranges[3][1], ranges
    assert any(a == b for a, b in ranges[1:3]), ranges
    _run(case, X, (4,), 5, 10, pps=("l3-hinge", "log-l2-hinge"))


# ------------------------------------------------------------------------------------------------ tiles
def test_sharded_call_tiles(tmp_path, gpu_clib, monkeypatch):
    """PB200_WORKSPACE_MB=64 cuts 4,000 queries at beam 64 into several tiles: every rank's records and the merged result
    equal the one-tile call."""
    layers = random_tree(501, [64, 16384], 300, 20, bias=1.0)
    case = _Case(gpu_clib, _save(str(tmp_path / "m"), layers), layers)
    X = synth.make_queries(761, 4000, 300, 30)
    world = 3

    def launches():
        return sum(case.c.pb200_xlinear_launches(m.model_chain) for m in case.shards(world))

    monkeypatch.delenv("PB200_WORKSPACE_MB", raising=False)
    l0 = launches()
    want, w_sent, _ = case.sharded(X, world, 64, 10, None, 1)
    l1 = launches()
    monkeypatch.setenv("PB200_WORKSPACE_MB", "64")
    try:
        got, g_sent, _ = case.sharded(X, world, 64, 10, None, 1)
    finally:
        monkeypatch.delenv("PB200_WORKSPACE_MB", raising=False)
    l2 = launches()
    assert l2 - l1 > l1 - l0, f"{l2 - l1} launches at 64 MiB vs {l1 - l0} in one tile: the call was not tiled"
    assert want.nnz > 0
    _same_bits(got, want, "tiled vs one tile")
    for r in range(world):
        assert np.array_equal(g_sent[r].cpu().numpy(), w_sent[r].cpu().numpy()), f"rank {r}: tiled records differ"
    _same_bits(want, case.unsharded(X, 64, 10, None, 1), "one tile vs unsharded")


# ------------------------------------------------------------------------------------------------ capacity
@pytest.mark.parametrize("world,topk", [(2, 512), (4, 256), (8, 128)])
def test_xlinear_merge_capacity_is_reached(wide_leaf, world, topk):
    case, D = wide_leaf
    X = _queries(771, D, [40] * 60 + [100])
    assert world * case.clib.xlinear_plan_stride(case.h, 40, topk) == CAP
    _run(case, X, (world,), 40, topk, pps=("l3-hinge",), modes=(1, 0))


def test_narrow_stride_passes_where_k_would_not(wide_leaf):
    """World 8 and only_topk 200 at beam 2: a leaf row holds at most 2 x 64 = 128 candidates, so the stride is 128 and
    8 x 128 = 1,024 records fit, although 8 x 200 would not."""
    case, D = wide_leaf
    X = _queries(772, D, [40] * 60 + [100])
    assert case.clib.xlinear_plan_stride(case.h, 2, 200) == 128
    want = _run(case, X, (8,), 2, 200, pps=("l3-hinge",), modes=(1, 0))
    assert np.all(np.diff(want.indptr) == 128)


@pytest.mark.parametrize("world,topk", [(5, 205), (8, 129)])
def test_xlinear_past_the_merge_capacity_raises_before_gpu_work(wide_leaf, world, topk):
    case, D = wide_leaf
    X = _queries(773, D, [40] * 20)
    for m in case.shards(world):
        before = case.c.pb200_xlinear_launches(m.model_chain)
        m.comm.sent = None
        with pytest.raises(ValueError, match=f"world \\* top-k = {world * topk} exceeds the merge capacity of 1024"):
            m.predict(X, beam_size=40, only_topk=topk)
        assert case.c.pb200_xlinear_launches(m.model_chain) == before and m.comm.sent is None


@pytest.fixture(scope="module")
def hnsw_base():
    return hnsw_rows(781, 1600, 32, False), hnsw_rows(782, 150, 32, False)  # 150 queries: not a multiple of 4


@pytest.mark.parametrize("world,topk,efS", [(8, 128, 160), (2, 512, 600)])
def test_hnsw_merge_capacity_is_reached(tmp_path, gpu_clib, hnsw_base, world, topk, efS):
    from pecos_b200.hnsw_build import build_hnsw_shards

    X, Q = hnsw_base
    folder = str(tmp_path / "s")
    build_hnsw_shards(X, folder, world, seed=5, M=8, efC=40, metric="l2", device="cuda:0")
    got, want, s0 = _hnsw_sharded_predict(folder, Q, efS, topk)
    _bits_equal(got, want, f"world={world} topk={topk}")
    keys, _, _ = _records(s0.comm.parts[world - 1])
    # the last rank's last slot: low word ~(rank * topk + slot) = ~1023
    assert np.all(keys[:, -1] & np.uint64(0xFFFFFFFF) == np.uint64(0xFFFFFFFF - (CAP - 1)))


def test_hnsw_past_the_merge_capacity_is_refused_before_any_launch(tmp_path, gpu_clib, hnsw_base):
    from pecos_b200.distributed import ShardedHNSW
    from pecos_b200.hnsw import HNSW
    from pecos_b200.hnsw_build import build_hnsw_shards

    X, Q = hnsw_base
    folder = str(tmp_path / "s")
    build_hnsw_shards(X, folder, 5, seed=6, M=8, efC=40, metric="l2", device="cuda:0")
    for r in range(5):
        s = ShardedHNSW.load(folder, comm=_StackComm(r, 5))
        out = (c_uint64 * 8)()
        gpu_clib.clib_float32.pb200_hnsw_get_info(s.index.model_ptr, out)
        before = int(out[7])
        with pytest.raises(ValueError, match="world \\* topk = 1025 exceeds the merge capacity of 1024"):
            s.predict(Q, HNSW.PredParams(efS=300, topk=205))
        gpu_clib.clib_float32.pb200_hnsw_get_info(s.index.model_ptr, out)
        assert int(out[7]) == before and s.comm.sent is None


# ------------------------------------------------------------------------------------------------ coverage (keep last)
def test_every_leaf_kernel_ran_on_a_rank_with_absent_chunks():
    """The cases above ran each of these on a rank that does not own every leaf chunk."""
    need = {"score 0", "score 1", "score 3", "score 4", "prefix", "block top-k, one sort", "block top-k, streaming",
            "warp select, k > 32", "estimate filter"}
    missing = need - _SEEN
    assert not missing, f"not seen on a sharded leaf: {sorted(missing)}; seen: {sorted(_SEEN)}"
