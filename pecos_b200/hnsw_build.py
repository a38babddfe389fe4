"""GPU construction of an HNSW index in the reference's on-disk format (SURVEY 8f-4).

What it replaces: ``HNSW::train`` (pecos/core/ann/hnsw.hpp:677-846), the reference's incremental, lock-based CPU build
(44 s for 100k x 768, 797 s for 1M x 768 on 128 host threads) -- the step that kept BASELINE.json's 10M-vector configuration
out of reach.  What it produces: ``<folder>/param.json`` + ``<folder>/c_model/{config.json, index.mmap_store}``, byte-compatible
with what ``HNSW.save`` writes (hnsw.hpp:490-532, GraphL0 :104-120, GraphL1 :188-219, container pecos/core/utils/mmap_util.hpp),
so BOTH the reference library and pecos_b200 load and search it.

Parity contract (VERDICT r1, item 9): the BUILD is recall-level -- a batch construction cannot reproduce the insertion-order
dependent graph of the incremental algorithm (the reference itself is nondeterministic with threads > 1, hnsw.hpp:804-809);
SEARCH on the saved file is bit-level: the reference and the CUDA engine return identical ids / distance bits on it
(tests/test_hnsw_build_gpu.py).

Both index kinds are built: dense (``drm``, float32 rows) and sparse (``csr``, a scipy sparse matrix).  Only the two distance
computations differ; levels, the prefix kNN, the heuristic, reverse links and the records' order are shared:

* dense: the distance work is dense GEMMs on the tensor cores, cuBLAS through torch -- a plain library GEMM -- instead of
  10^9 dependent single-vector distance calls;
* sparse: the project's kernels in csrc/hnsw_build_sparse.cu (an inverted-index block kernel for the prefix kNN, a
  sorted-merge kernel for the heuristic's candidate sets).  Every distance is bit-identical to the reference's
  FeatVecSparse{IP,L2}Simd::distance (ip: 1 - <x,y>; l2: the reference's -2<x,y>), so neighbours are ranked and the
  heuristic decides by exactly the distances the search and the reference's own train use.  On ``device="cpu"`` the sparse
  distances are scipy products instead (tiny inputs only).

Algorithm:

1. node levels as the reference draws them: ``floor(-ln(U) / ln(M))`` (hnsw.hpp:785-793), entry point = first node of the top level;
2. for every level l and node i: the EXACT k = efC nearest among the nodes present at l that the incremental algorithm would
   already have inserted (ids < i; hnsw.hpp:804-809 inserts in id order), by tiled brute force (``X_tile @ X^T`` over the lower
   triangle + running top-k) -- the prefix constraint gives early nodes their long-range links, i.e. the navigability of the
   incrementally built graph;
3. the reference's neighbour-selection heuristic (hnsw.hpp:556-592: keep a candidate iff it is closer to the node than to
   every neighbour kept so far; at most M; fewer than M candidates are kept whole), evaluated for a whole tile of nodes at
   once from the candidates' pairwise distance matrix (one batched GEMM, or the candidate-set kernel);
4. reverse links: every selected edge u -> v also offers u to v; a node whose selected + offered set exceeds the level's
   capacity (maxM0 = 2M at level 0, maxM above) is pruned with the same heuristic (hnsw.hpp:628-652);
5. neighbour lists sorted by ascending distance (hnsw.hpp:823-845), records laid out as GraphL0 / GraphL1 store them
   (sparse GraphL0 records are variable-size FeatVecSparse records located by byte offsets).

torch is used for device memory and the GEMM / top-k primitives; nothing here is on the search path.

``build_hnsw_shards`` splits the rows into contiguous ranges and builds one such index per range (an index larger than one GPU,
built in parallel on several); ``pecos_b200.distributed.ShardedHNSW`` searches it.
"""
import contextlib
import json
import math
import os
import time

import numpy as np

_HNSW_T = {
    "ip": "pecos::ann::HNSW<float, pecos::ann::FeatVecDenseIPSimd<float>>",
    "l2": "pecos::ann::HNSW<float, pecos::ann::FeatVecDenseL2Simd<float>>",
}
_HNSW_T_SPARSE = {
    "ip": "pecos::ann::HNSW<float, pecos::ann::FeatVecSparseIPSimd<uint32_t, float>>",
    "l2": "pecos::ann::HNSW<float, pecos::ann::FeatVecSparseL2Simd<uint32_t, float>>",
}
_SPARSE_CAND_MAX = 512        # widest candidate set of the candidate-set kernel (kCandMax in csrc/hnsw_build_sparse.cu)
_SPARSE_C_TILE_MAX = 24576    # block-kernel accumulators that fit its shared-memory budget (kAccSmemMax / 4)


# ------------------------------------------------------------------------------------------------ container writer
def write_mmap_store(path, blocks):
    """PECOS MmapStore container (pecos/core/utils/mmap_util.hpp:54-184): data blocks, each padded to 16-byte alignment,
    then the metadata ``[n_blocks u64][(offset u64, size u64) x n]``, then the 16-byte signature
    ``0x93 'PECOS' | '<' | version 1 | metadata offset u64``.  ``blocks``: list of bytes-like / numpy arrays."""
    info = []
    with open(path, "wb") as f:
        off = 0
        for b in blocks:
            raw = b.tobytes() if isinstance(b, np.ndarray) else bytes(b)
            info.append((off, len(raw)))
            f.write(raw)
            off += len(raw)
            pad = (-off) % 16
            if pad:
                f.write(b"\0" * pad)
                off += pad
        meta = np.array([len(info)] + [v for pair in info for v in pair], dtype="<u8").tobytes()
        f.write(meta)
        f.write(b"\x93PECOS" + b"<" + bytes([1]) + np.array([off], dtype="<u8").tobytes())


def _scalar(v, dtype="<u4"):
    return np.array([v], dtype=dtype)


def _vector(arr):
    """MmapableVector = two blocks: size u64, then the elements (mmap_util.hpp:526-537)."""
    arr = np.ascontiguousarray(arr)
    return [np.array([arr.size], dtype="<u8"), arr]


# ------------------------------------------------------------------------------------------------ distance helpers
def _pairwise(torch, A, B, metric, a_sq=None, b_sq=None):
    """distance(A_i, B_j): ip -> 1 - <a, b>; l2 -> |a|^2 + |b|^2 - 2<a, b> (clamped at 0)."""
    G = A @ B.transpose(-1, -2)
    if metric == "ip":
        return 1.0 - G
    if a_sq is None:
        a_sq = (A * A).sum(-1)
    if b_sq is None:
        b_sq = (B * B).sum(-1)
    return (a_sq.unsqueeze(-1) + b_sq.unsqueeze(-2) - 2.0 * G).clamp_min_(0.0)


class _PhaseTimer(object):
    """Build time per phase: CUDA events on the current stream (read once, at the end) or a host clock on the CPU."""

    def __init__(self, torch, dev):
        self.torch, self.cuda = torch, dev.type == "cuda"
        self.marks = {}

    @contextlib.contextmanager
    def __call__(self, name):
        if self.cuda:
            a, b = self.torch.cuda.Event(enable_timing=True), self.torch.cuda.Event(enable_timing=True)
            a.record()
            yield
            b.record()
        else:
            a = time.perf_counter()
            yield
            b = time.perf_counter()
        self.marks.setdefault(name, []).append((a, b))

    def totals_ms(self):
        if self.cuda:
            self.torch.cuda.synchronize()
            return {k: float(sum(a.elapsed_time(b) for a, b in v)) for k, v in self.marks.items()}
        return {k: float(sum(b - a for a, b in v) * 1e3) for k, v in self.marks.items()}


def _dense_distances(torch, X, metric):
    """The two distance functions of a dense build: (block_for(ids) -> block(q0, q1, c0, c1), cand_dist(cand))."""
    sq = (X * X).sum(-1) if metric == "l2" else None

    def block_for(ids):
        def block(q0, q1, c0, c1):
            qi, ci = ids[q0:q1], ids[c0:c1]
            return _pairwise(torch, X[qi], X[ci], metric, None if sq is None else sq[qi], None if sq is None else sq[ci])
        return block

    def cand_dist(c):
        V = X[c.clamp_min(0)]                                   # [T, C, d]
        return _pairwise(torch, V, V, metric)                   # [T, C, C] candidate-to-candidate distances

    return block_for, cand_dist


def _finalize_sparse_np(dot, metric):
    """FeatVecSparse{IP,L2}Simd::distance from float32 dot products: 1 - dot, or -2 dot (the reference's sparse "l2")."""
    dot = dot.astype(np.float64)
    return ((1.0 - dot) if metric == "ip" else (0.0 - 2.0 * dot)).astype(np.float32)


def _sparse_distances_cpu(torch, Xc, metric):
    """Sparse distance functions on the CPU (scipy products; small inputs, e.g. format tests on a box without a GPU)."""

    def block_for(ids):
        idn = ids.numpy()

        def block(q0, q1, c0, c1):
            dot = (Xc[idn[q0:q1]] @ Xc[idn[c0:c1]].T).toarray().astype(np.float32)
            return torch.from_numpy(_finalize_sparse_np(dot, metric))
        return block

    def cand_dist(c):
        cn = c.numpy()
        T, C = cn.shape
        out = np.full((T, C, C), np.inf, dtype=np.float32)
        for t in range(T):
            ok = np.nonzero(cn[t] >= 0)[0]
            V = Xc[cn[t, ok]]
            out[t][np.ix_(ok, ok)] = _finalize_sparse_np((V @ V.T).toarray().astype(np.float32), metric)
        return torch.from_numpy(out)

    return block_for, cand_dist


class _SparseDevice(object):
    """Sparse distance functions on a CUDA device: the pb200_sparse_* kernels (csrc/hnsw_build_sparse.cu) over the rows in HBM
    as row_ptr (u64) + 8-byte {u32 index, f32 value} entries.  `work` counts what the kernels walked: [0] postings of the
    block kernel, [1] row entries of the candidate-set intersections."""

    def __init__(self, torch, Xc, metric, dev):
        from .core import get_clib

        self.torch, self.dev, self.metric = torch, dev, 0 if metric == "ip" else 1
        self.lib = get_clib().clib_float32
        self.D = Xc.shape[1]
        ent = np.empty((Xc.nnz, 2), dtype=np.uint32)
        ent[:, 0] = Xc.indices
        ent[:, 1] = Xc.data.view(np.uint32)
        self.row_ptr = torch.from_numpy(Xc.indptr.astype(np.int64)).to(dev)
        self.ent = torch.from_numpy(ent.view(np.int32)).to(dev)          # [nnz, 2]
        self.work = torch.zeros(2, dtype=torch.int64, device=dev)

    def _stream(self):
        return self.torch.cuda.current_stream(self.dev).cuda_stream

    def block_for(self, ids):
        """Inverted index of the level's rows (positions into ids, ascending within a column) and the block function."""
        torch = self.torch
        starts, lens = self.row_ptr[ids], self.row_ptr[ids + 1] - self.row_ptr[ids]
        pos = torch.repeat_interleave(torch.arange(ids.numel(), device=self.dev), lens)
        first = torch.cumsum(lens, 0) - lens
        src = torch.arange(pos.numel(), device=self.dev) - first[pos] + starts[pos]
        e = self.ent[src]
        col = e[:, 0].long()
        order = torch.argsort(col, stable=True)                           # stable: positions stay ascending per column
        post = torch.stack([pos[order].int(), e[order, 1]], 1).contiguous()
        col_ptr = torch.zeros(self.D + 1, dtype=torch.int64, device=self.dev)
        col_ptr[1:] = torch.cumsum(torch.bincount(col, minlength=self.D), 0)
        del starts, lens, pos, first, src, e, col, order
        ids = ids.contiguous()

        def block(q0, q1, c0, c1):
            out = torch.empty((q1 - q0, c1 - c0), dtype=torch.float32, device=self.dev)
            self.lib.pb200_sparse_block_distances(self.dev.index, self.metric, self.row_ptr.data_ptr(), self.ent.data_ptr(),
                                                  ids[q0:q1].data_ptr(), q1 - q0, col_ptr.data_ptr(), post.data_ptr(), c0, c1 - c0,
                                                  out.data_ptr(), self.work.data_ptr(), self._stream())
            return out
        return block

    def cand_dist(self, c):
        c = c.contiguous()
        T, C = c.shape
        out = self.torch.empty((T, C, C), dtype=self.torch.float32, device=self.dev)
        self.lib.pb200_sparse_candidate_distances(self.dev.index, self.metric, self.row_ptr.data_ptr(), self.ent.data_ptr(),
                                                  c.data_ptr(), T, C, out.data_ptr(), self.work.data_ptr() + 8, self._stream())
        return out


def _exact_knn(torch, block, n, k, q_tile, c_tile, dev, timer):
    """For every position 0..n-1 of a level's node list (ascending = the reference's insertion order): its k nearest EARLIER
    nodes -- what an incremental insertion can link a new node to (hnsw.hpp:742-760: the graph only holds the nodes inserted so
    far).  This prefix constraint is what makes the graph navigable: early nodes get long-range links, exactly as in the
    incremental algorithm (an unconstrained kNN graph has none: recall 0.89 at N = 20k, measured).  block(q0, q1, c0, c1):
    the distances between positions [q0, q1) and [c0, c1).  Returns (nbr positions [n, k], distances [n, k]) ascending;
    missing slots hold -1 / inf."""
    k = min(k, max(n - 1, 0))
    out_i = torch.full((n, max(k, 1)), -1, dtype=torch.long, device=dev)
    out_d = torch.full((n, max(k, 1)), float("inf"), dtype=torch.float32, device=dev)
    if k == 0:
        return out_i[:, :0], out_d[:, :0]
    for q0 in range(0, n, q_tile):
        q1 = min(n, q0 + q_tile)
        best_d = torch.full((q1 - q0, k), float("inf"), dtype=torch.float32, device=dev)
        best_i = torch.full((q1 - q0, k), -1, dtype=torch.long, device=dev)
        for c0 in range(0, q1, c_tile):                      # only earlier nodes can be candidates
            c1 = min(q1, c0 + c_tile)
            with timer("knn_distances"):
                D = block(q0, q1, c0, c1)
            with timer("knn_topk"):
                if c1 > q0:  # the tile reaches into the query rows' own range: keep strictly earlier positions only
                    rows = torch.arange(q0, q1, device=dev).unsqueeze(1)
                    cols = torch.arange(c0, c1, device=dev).unsqueeze(0)
                    D = torch.where(cols < rows, D, torch.full_like(D, float("inf")))
                cat_d = torch.cat([best_d, D], dim=1)
                cat_i = torch.cat([best_i, torch.arange(c0, c1, device=dev).expand(q1 - q0, -1)], dim=1)
                best_d, sel = torch.topk(cat_d, k, dim=1, largest=False, sorted=True)
                best_i = torch.gather(cat_i, 1, sel)
        out_d[q0:q1, :k] = best_d
        out_i[q0:q1, :k] = torch.where(torch.isinf(best_d), torch.full_like(best_i, -1), best_i)
    return out_i[:, :k], out_d[:, :k]


def _heuristic(torch, cand_dist, cand, cand_d, cap, tile):
    """The reference's get_neighbors_heuristic (hnsw.hpp:556-592) for many nodes at once.
    cand [n, C]: candidate ids (global), ascending by cand_d (distance to the node), -1 = empty; cand_dist(cand tile) -> the
    [T, C, C] candidate-to-candidate distances.  Returns kept mask [n, C]:
    a node with fewer than `cap` candidates keeps all of them; else candidates are visited in order and kept iff no
    already-kept candidate is strictly closer to them than the node is, until `cap` are kept."""
    n, C = cand.shape
    dev = cand.device
    kept_all = torch.zeros((n, C), dtype=torch.bool, device=dev)
    valid_all = cand >= 0
    for t0 in range(0, n, tile):
        t1 = min(n, t0 + tile)
        c = cand[t0:t1]
        valid = valid_all[t0:t1]
        dq = cand_d[t0:t1]
        D = cand_dist(c)
        few = valid.sum(1) < cap
        kept = torch.zeros_like(valid)
        count = torch.zeros(t1 - t0, dtype=torch.long, device=dev)
        for j in range(C):
            bad = ((D[:, :, j] < dq[:, j:j + 1]) & kept).any(dim=1)
            ok = valid[:, j] & ~bad & (count < cap)
            kept[:, j] = ok
            count += ok.long()
        kept_all[t0:t1] = torch.where(few.unsqueeze(1), valid, kept)
    return kept_all


def _build_level(torch, ids, M, cap, efC, block_for, cand_dist, q_tile, c_tile, h_tile, timer):
    """Neighbour lists (global ids, ascending distance, <= cap each) of the nodes `ids` on one level.  block_for(ids) -> the
    level's block-distance function (see _exact_knn); cand_dist: candidate-set distances (see _heuristic)."""
    n = ids.numel()
    dev = ids.device
    lists = torch.full((n, cap), -1, dtype=torch.long, device=dev)
    if n <= 1:
        return lists, torch.zeros(n, dtype=torch.long, device=dev)
    with timer("knn_distances"):
        block = block_for(ids)
    pos, dist = _exact_knn(torch, block, n, efC, q_tile, c_tile, dev, timer)   # positions into ids
    del block
    cand = torch.where(pos >= 0, ids[pos.clamp_min(0)], torch.full_like(pos, -1))
    with timer("heuristic"):
        keep = _heuristic(torch, cand_dist, cand, dist, M, h_tile)             # forward selection: at most M (hnsw.hpp:598)
    with timer("reverse_links"):
        pool, pool_d, counts = _reverse_pools(torch, ids, pos, dist, cand, keep, cap)
    over = counts > cap
    keep2 = pool >= 0
    if bool(over.any()):
        idx = torch.nonzero(over).squeeze(1)
        with timer("heuristic"):
            keep2[idx] = _heuristic(torch, cand_dist, pool[idx], pool_d[idx], cap, h_tile)
    with timer("reverse_links"):
        # compact the kept neighbours (already ascending by distance)
        rank2 = torch.cumsum(keep2.long(), 1) - 1
        rows = torch.arange(n, device=dev).unsqueeze(1).expand_as(pool)
        sel = keep2 & (rank2 < cap)
        lists[rows[sel], rank2[sel]] = pool[sel]
    return lists, sel.sum(1)


def _reverse_pools(torch, ids, pos, dist, cand, keep, cap):
    """Every node's pool = its selected neighbours + the nodes that selected it, ascending by distance, truncated to a working
    width.  Returns (pool ids [n, width], distances, pool sizes before truncation)."""
    n = ids.numel()
    dev = ids.device
    # edges u -> v (selected) and the offers v <- u
    src = torch.arange(n, device=dev).unsqueeze(1).expand_as(cand)[keep]       # positions
    dst_pos = pos[keep]
    d_uv = dist[keep]
    # every node's pool = its selected + the nodes that selected it; dedupe (u, v) pairs
    a = torch.cat([src, dst_pos])
    b = torch.cat([dst_pos, src])
    d = torch.cat([d_uv, d_uv])
    key = a * n + b
    order = torch.argsort(key, stable=True)
    key, a, b, d = key[order], a[order], b[order], d[order]
    first = torch.ones_like(key, dtype=torch.bool)
    first[1:] = key[1:] != key[:-1]
    a, b, d = a[first], b[first], d[first]
    # per node: pool sorted by distance, truncated to a working width (the heuristic only ever needs the closest few)
    width = min(max(4 * cap, 64), 512)
    order = torch.argsort(d, stable=True)
    a, b, d = a[order], b[order], d[order]
    order = torch.argsort(a, stable=True)
    a, b, d = a[order], b[order], d[order]
    counts = torch.bincount(a, minlength=n)
    starts = torch.cumsum(counts, 0) - counts
    rank = torch.arange(a.numel(), device=dev) - starts[a]
    ok = rank < width
    pool = torch.full((n, width), -1, dtype=torch.long, device=dev)
    pool_d = torch.full((n, width), float("inf"), dtype=torch.float32, device=dev)
    pool[a[ok], rank[ok]] = ids[b[ok]]
    pool_d[a[ok], rank[ok]] = d[ok]
    return pool, pool_d, counts


# ------------------------------------------------------------------------------------------------ public entry point
def _pred_kwargs(pred_kwargs):
    pk = {"efS": 100, "topk": 10, "threads": 1}
    pk.update(pred_kwargs or {})
    return pk


def build_hnsw_index(X, folder, M=32, efC=100, metric="ip", seed=0, max_level_upper_bound=-1, device=None, pred_kwargs=None,
                     q_tile=4096, c_tile=65536, h_tile=None, allow_tf32=False):
    """Builds the index for the rows of ``X`` and writes it to ``folder`` in the reference's format.  ``X``: float32 [N, d]
    (a dense ``drm`` index) or a scipy sparse matrix (a sparse ``csr`` index: converted to float32 csr and canonicalised with
    ``sum_duplicates()`` / ``sort_indices()``; the canonical rows are stored; efC <= 512; c_tile is capped at 24,576 so the
    block kernel's accumulators stay in shared memory).  Returns a dict with the build statistics, including the build time
    per phase (``phase_ms``).  ``device``: torch device (default: cuda:0; "cpu" is accepted for tiny inputs, e.g. format
    tests on a box without a GPU)."""
    import scipy.sparse as smat
    import torch

    if metric not in _HNSW_T:
        raise ValueError(f"metric must be 'ip' or 'l2', got {metric!r}")
    sparse = smat.issparse(X)
    if sparse:
        X = smat.csr_matrix(X, dtype=np.float32, copy=True)
        X.sum_duplicates()
        X.sort_indices()
        if int(efC) > _SPARSE_CAND_MAX:
            raise ValueError(f"efC must be <= {_SPARSE_CAND_MAX} for csr input, got {efC}")
        c_tile = min(int(c_tile), _SPARSE_C_TILE_MAX)
    else:
        X = np.ascontiguousarray(X, dtype=np.float32)
    N, d = X.shape
    if N < 1:
        raise ValueError("empty input")
    dev = torch.device(device if device is not None else "cuda:0")
    if dev.type == "cuda":
        dev = torch.device("cuda", dev.index if dev.index is not None else torch.cuda.current_device())
        torch.backends.cuda.matmul.allow_tf32 = bool(allow_tf32)
    timer = _PhaseTimer(torch, dev)
    maxM, maxM0 = int(M), 2 * int(M)
    if h_tile is None:  # the [T, C, C] candidate distances (+ the gathered [T, C, d] rows of a dense build) within 256 MB
        h_tile = max(16, min(2048, (256 << 20) // (4 * max(4 * maxM0, 64) * max(4 * maxM0, 64, 0 if sparse else d))))

    # 1. levels (hnsw.hpp:785-793) and the entry point
    rng = np.random.default_rng(seed)
    u = 1.0 - rng.random(N)  # (0, 1]
    levels = np.floor(-np.log(u) * (1.0 / math.log(float(maxM)))).astype(np.int64)
    if max_level_upper_bound >= 0:
        levels = np.minimum(levels, int(max_level_upper_bound))
    max_level = int(levels.max())
    init_node = int(np.argmax(levels == max_level))

    with timer("upload"):
        if not sparse:
            block_for, cand_dist = _dense_distances(torch, torch.from_numpy(X).to(dev), metric)
        elif dev.type == "cuda":
            sp = _SparseDevice(torch, X, metric, dev)
            block_for, cand_dist = sp.block_for, sp.cand_dist
        else:
            block_for, cand_dist = _sparse_distances_cpu(torch, X, metric)
        lvl = torch.from_numpy(levels).to(dev)
    level_lists = []
    for l in range(0, max_level + 1):
        ids = torch.nonzero(lvl >= l).squeeze(1)
        cap = maxM0 if l == 0 else maxM
        lists, deg = _build_level(torch, ids, maxM, cap, int(efC), block_for, cand_dist, q_tile, c_tile, h_tile, timer)
        with timer("download"):
            level_lists.append((ids.cpu().numpy(), lists.cpu().numpy(), deg.cpu().numpy()))

    t0 = time.perf_counter()
    # 2. records.  GraphL0: per node [deg u32][maxM0 ids u32][feature vector] (hnsw.hpp:47-91, :104-178)
    ids0, lists0, deg0 = level_lists[0]
    head = np.zeros((N, 1 + maxM0), dtype="<u4")
    head[ids0, 0] = deg0
    nb = np.where(lists0 >= 0, lists0, 0).astype("<u4")
    head[ids0, 1:] = nb
    if sparse:
        rec, mem_start, l0 = _sparse_records(head, X)
    else:
        # dense vector: [len u32][d f32]
        rec = 4 * (1 + maxM0) + 4 + 4 * d
        l0 = np.zeros((N, rec), dtype=np.uint8)
        l0[:, : 4 * (1 + maxM0)] = head.view(np.uint8)
        l0[:, 4 * (1 + maxM0): 4 * (1 + maxM0) + 4] = np.full((N, 1), d, dtype="<u4").view(np.uint8)
        l0[:, 4 * (1 + maxM0) + 4:] = X.view(np.uint8).reshape(N, 4 * d)
        mem_start = (np.arange(N + 1, dtype="<u8") * rec)
    # GraphL1: per node max_level slots of [deg u32][maxM ids u32] (hnsw.hpp:188-219); every node gets all slots
    level_mem = 1 + maxM
    node_mem = max_level * level_mem
    l1 = np.zeros(N * node_mem, dtype="<u4")
    for l in range(1, max_level + 1):
        ids_l, lists_l, deg_l = level_lists[l]
        base = ids_l.astype(np.int64) * node_mem + (l - 1) * level_mem
        l1[base] = deg_l
        cols = np.where(lists_l >= 0, lists_l, 0).astype("<u4")
        l1[(base[:, None] + 1 + np.arange(maxM)[None, :]).ravel()] = cols.ravel()

    # 3. files
    c_model = os.path.join(folder, "c_model")
    os.makedirs(c_model, exist_ok=True)
    blocks = [_scalar(N), _scalar(maxM), _scalar(maxM0), _scalar(int(efC)), _scalar(max_level), _scalar(init_node),
              _scalar(N), _scalar(d), _scalar(maxM0), _scalar(rec)] + _vector(mem_start) + _vector(l0.reshape(-1)) + \
             [_scalar(N), _scalar(max_level), _scalar(maxM), _scalar(node_mem), _scalar(level_mem)] + _vector(l1)
    write_mmap_store(os.path.join(c_model, "index.mmap_store"), blocks)
    with open(os.path.join(c_model, "config.json"), "w", encoding="utf-8") as f:
        json.dump({"hnsw_t": (_HNSW_T_SPARSE if sparse else _HNSW_T)[metric], "version": "v2.0",
                   "train_params": {"num_node": N, "maxM": maxM, "maxM0": maxM0, "efC": int(efC), "max_level": max_level,
                                    "init_node": init_node}}, f, indent=4)
    with open(os.path.join(folder, "param.json"), "w", encoding="utf-8") as f:
        json.dump({"model": "HNSW", "data_type": "csr" if sparse else "drm", "metric_type": metric, "num_item": N, "feat_dim": d,
                   "train_kwargs": {"M": maxM, "efC": int(efC), "builder": "pecos_b200.hnsw_build (batch, exact kNN + heuristic)"},
                   "pred_kwargs": _pred_kwargs(pred_kwargs)}, f, indent=1)
    phase_ms = timer.totals_ms()
    phase_ms["write"] = (time.perf_counter() - t0) * 1e3
    stats = {"num_node": N, "feat_dim": d, "max_level": max_level, "init_node": init_node,
             "mean_degree_l0": float(deg0.mean()), "nodes_per_level": [int(t[0].size) for t in level_lists], "phase_ms": phase_ms}
    if sparse and dev.type == "cuda":
        work = sp.work.cpu().tolist()
        stats["block_postings"], stats["candidate_entries"] = int(work[0]), int(work[1])
    return stats


SHARDS_MANIFEST = "shards.json"


def build_hnsw_shards(X, folder, world, ranks=None, device=None, seed=0, **build_kwargs):
    """Builds a sharded index: the rows of ``X`` split into ``world`` contiguous ranges, one independent index per range in
    ``<folder>/shard-<r>/`` (an ordinary index folder written by :func:`build_hnsw_index` with seed ``seed + r``), and the
    manifest ``<folder>/shards.json``.  Shard r's node j is global id ``row_begin[r] + j``.  Ranges: equal row counts for dense
    ``X``, ``distributed.split_rows_by_nnz`` of the csr indptr for sparse ``X``.

    Only the shards listed in ``ranks`` (default: all) are built, so under torchrun every rank builds its own with
    ``ranks=[rank]`` on its GPU.  The manifest depends only on X's shape (or indptr), ``world``, ``seed`` and the build
    arguments, so every caller writes the same file.  ``pecos_b200.distributed.ShardedHNSW`` searches the result.  Returns
    ``{"manifest": ..., "shards": {rank: build statistics}}``."""
    import scipy.sparse as smat

    from .distributed import split_rows_by_nnz

    world = int(world)
    if world < 1:
        raise ValueError(f"world must be >= 1, got {world}")
    ranks = list(range(world)) if ranks is None else [int(r) for r in ranks]
    if any(r < 0 or r >= world for r in ranks):
        raise ValueError(f"ranks {ranks} are outside 0..{world - 1}")
    sparse = smat.issparse(X)
    if sparse:
        X = smat.csr_matrix(X)
        row_begin = [int(b) for b in split_rows_by_nnz(X.indptr, world)]
    else:
        X = np.ascontiguousarray(X, dtype=np.float32)
        row_begin = [X.shape[0] * r // world for r in range(world + 1)]
    if any(row_begin[r + 1] <= row_begin[r] for r in range(world)):
        raise ValueError(f"{X.shape[0]} rows cannot fill {world} non-empty shards (row ranges {row_begin})")
    manifest = {"world": world, "num_item": int(X.shape[0]), "feat_dim": int(X.shape[1]), "data_type": "csr" if sparse else "drm",
                "metric_type": build_kwargs.get("metric", "ip"), "row_begin": row_begin,
                "seeds": [int(seed) + r for r in range(world)], "pred_kwargs": _pred_kwargs(build_kwargs.get("pred_kwargs"))}
    shards = {}
    for r in ranks:
        shards[r] = build_hnsw_index(X[row_begin[r]:row_begin[r + 1]], os.path.join(folder, f"shard-{r}"), seed=int(seed) + r,
                                     device=device, **build_kwargs)
    os.makedirs(folder, exist_ok=True)
    tmp = os.path.join(folder, f".{SHARDS_MANIFEST}.{os.getpid()}")
    with open(tmp, "w", encoding="utf-8") as f:
        json.dump(manifest, f, indent=1)
    os.replace(tmp, os.path.join(folder, SHARDS_MANIFEST))  # atomic: concurrent writers leave one complete copy
    return {"manifest": manifest, "shards": shards}


def _sparse_records(head, X):
    """GraphL0 records of a csr index (hnsw.hpp:92-178, FeatVecSparse feat_vectors.hpp:100-131): per node
    [deg u32][maxM0 ids u32][len u32][len f32 values][len u32 indices], variable size, located by mem_start_of_node (the byte
    offsets' prefix sum); the fixed record size is written as 0, as the reference does.  Returns (0, mem_start, buffer)."""
    N, h = head.shape
    lens = np.diff(X.indptr).astype(np.int64)
    sizes = 4 * (h + 1) + 8 * lens
    mem_start = np.zeros(N + 1, dtype="<u8")
    np.cumsum(sizes, out=mem_start[1:])
    buf = np.zeros(int(mem_start[-1]) // 4, dtype="<u4")
    base = mem_start[:-1].astype(np.int64) // 4
    buf[(base[:, None] + np.arange(h)[None, :]).ravel()] = head.ravel()
    buf[base + h] = lens
    first = np.repeat(base + h + 1 - X.indptr[:-1].astype(np.int64), lens) + np.arange(X.nnz, dtype=np.int64)
    buf[first] = X.data.view("<u4")
    buf[first + np.repeat(lens, lens)] = X.indices.astype("<u4")
    return 0, mem_start, buf.view(np.uint8)
