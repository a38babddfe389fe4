"""Helpers of the HNSW index-sharding tests (test infrastructure): query/base rows with non-zero distances, the key rule of
the exchange records restated in numpy, and the numpy merge of per-shard search results."""
import numpy as np
import scipy.sparse as smat

from .util import merge_shards_numpy


def hnsw_rows(seed, n, d, sparse):
    """Base or query rows for the HNSW sharding tests: dense unit float32 rows, or csr rows (about 8 entries) that all hold
    column 0 with a positive value, so that every query/row distance is non-zero for both metrics (the reference's sparse "l2"
    is -2<x,y>: 0.0 for rows without a common column)."""
    rng = np.random.default_rng(seed)
    if not sparse:
        X = rng.standard_normal((n, d)).astype(np.float32)
        return X / np.linalg.norm(X, axis=1, keepdims=True)
    M = smat.random(n, d - 1, density=min(1.0, 7.0 / (d - 1)), format="csr", dtype=np.float32, random_state=rng)
    M.data[:] = rng.random(M.nnz).astype(np.float32) + np.float32(0.1)
    X = smat.hstack([smat.csr_matrix((rng.random(n).astype(np.float32) + np.float32(0.1))[:, None]), M], format="csr")
    X.sort_indices()
    return X.astype(np.float32)


def hnsw_result_counts(idx, dist):
    """Filled slots per row of a zero-filled HNSW result (rows x topk): a row ends after its last slot that is not (id 0,
    distance bits 0).  Exact as long as no real neighbour is node 0 at distance +0.0 (hnsw_rows guarantees non-zero distances)."""
    filled = ~((idx == 0) & (np.asarray(dist, dtype=np.float32).view(np.uint32) == 0))
    rev = filled[:, ::-1]
    return np.where(rev.any(1), idx.shape[1] - rev.argmax(1), 0).astype(np.uint32)


def hnsw_shard_records(idx, dist, cnt, rank, id_offset, topk):
    """One shard's exchange records (test-only restatement of hnsw_shard_pack_kernel): (keys u64, global ids, distances)
    rows x topk, key = (~orderable(dist) << 32) | ~(rank * topk + slot), 0 for the slots at or beyond cnt; every NaN, whatever
    its sign and payload, has orderable 0xFFFFFFFF (after +inf)."""
    u = np.asarray(dist, dtype=np.float32).view(np.uint32).astype(np.uint64)
    order = np.where(u & np.uint64(0x80000000), ~u & np.uint64(0xFFFFFFFF), u | np.uint64(0x80000000))
    order = np.where(np.isnan(np.asarray(dist, dtype=np.float32)), np.uint64(0xFFFFFFFF), order)
    low = ~(np.uint64(rank * topk) + np.arange(topk, dtype=np.uint64)) & np.uint64(0xFFFFFFFF)
    keys = ((~order & np.uint64(0xFFFFFFFF)) << np.uint64(32)) | low[None, :]
    valid = np.arange(topk)[None, :] < np.asarray(cnt)[:, None]
    keys = np.where(valid, keys, np.uint64(0))
    ids = np.where(valid, idx.astype(np.uint64) + np.uint64(id_offset), 0).astype(np.uint32)
    return keys, ids, np.where(valid, dist, np.float32(0)).astype(np.float32)


def merge_hnsw_shards_numpy(idx, dist, row_begin, topk):
    """Reference semantics of the HNSW shard merge (test-only): per-shard search results idx / dist [world][rows][topk]
    (local ids, zero-filled tails) -> the topk best of their union by (distance with NaN last, shard rank, slot), global ids
    row_begin[r] + local id, zero-filled tails.  Returns (ids, distances), rows x topk."""
    world = idx.shape[0]
    recs = [hnsw_shard_records(idx[r], dist[r], hnsw_result_counts(idx[r], dist[r]), r, row_begin[r], topk) for r in range(world)]
    keys, ids, vals = (np.stack([rc[i] for rc in recs]) for i in range(3))
    out_ids, out_vals, _ = merge_shards_numpy(keys, ids, vals, (keys != 0).sum(2), topk)
    return out_ids, out_vals


