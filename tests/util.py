"""Shared helpers for the parity tests (test infrastructure)."""
import os

import numpy as np
import scipy.sparse as smat

from pecos_b200 import synth


def assert_csr_parity(got, want, rtol=1e-5, what=""):
    """Bit-exact label ids and ranks (stored order), scores within `rtol` relative (BASELINE.json north_star)."""
    assert got.shape == want.shape, f"{what}: shape {got.shape} != {want.shape}"
    assert np.array_equal(np.asarray(got.indptr, dtype=np.int64), np.asarray(want.indptr, dtype=np.int64)), f"{what}: row sizes differ"
    gi, wi = np.asarray(got.indices, dtype=np.int64), np.asarray(want.indices, dtype=np.int64)
    if not np.array_equal(gi, wi):
        bad = np.nonzero(gi != wi)[0]
        row = np.searchsorted(got.indptr, bad[0], side="right") - 1
        raise AssertionError(
            f"{what}: {bad.size} label ids / ranks differ; first at row {row}: got {gi[got.indptr[row]:got.indptr[row+1]]} "
            f"want {wi[want.indptr[row]:want.indptr[row+1]]}; scores got {got.data[got.indptr[row]:got.indptr[row+1]]} "
            f"want {want.data[want.indptr[row]:want.indptr[row+1]]}"
        )
    gd, wd = np.asarray(got.data, dtype=np.float32), np.asarray(want.data, dtype=np.float32)
    denom = np.maximum(np.abs(wd), np.finfo(np.float32).tiny)
    rel = np.abs(gd.astype(np.float64) - wd.astype(np.float64)) / denom
    assert rel.size == 0 or rel.max() <= rtol, f"{what}: max relative score error {rel.max():.3e} > {rtol}"
    exact = float(np.mean(gd.view(np.uint32) == wd.view(np.uint32))) if gd.size else 1.0
    return exact


def assert_same_nan(got, want, what="", tags="IMDV"):
    """Arrays tagged by `tags` (PairwiseANN: I, M, D, V; HNSW: I, D) bit-equal, except that in D two NaNs of any payload
    are equal: the GPU returns 0x7FFFFFFF for every NaN, x86 the first NaN operand or 0xFFC00000."""
    for tag, g, w in zip(tags, got, want):
        g, w = np.asarray(g), np.asarray(w)
        if tag == "D":
            both = np.isnan(g) & np.isnan(w)
            assert np.array_equal(np.where(both, 0, g.view(np.uint32)), np.where(both, 0, w.view(np.uint32))), f"D {what}"
        else:
            assert np.array_equal(g.view(np.uint32), w.view(np.uint32)), f"{tag} {what}"


def random_tree(seed, layer_sizes, D, nnz_per_col, bias=1.0, permute=False, prune=0.0, saturate=False):
    """Random label tree; `permute` shuffles child->parent assignment (non-contiguous C), `prune` drops that fraction of
    rows from every non-root C (pruned tree, pecos set_output_constraint style), `saturate` scales weights up so that the
    hinge post-processors saturate and ties decide the ranking."""
    rng = np.random.default_rng(seed)
    layers = synth.make_tree_model(seed, layer_sizes, D, nnz_per_col, bias=bias)
    out = []
    for d, (W, C) in enumerate(layers):
        if saturate:
            W = W * np.float32(8.0)
        C = smat.csc_matrix(C)
        if permute and d > 0 and C.shape[0] > 1:
            perm = rng.permutation(C.shape[0])
            C = smat.csc_matrix(C.tocsr()[perm, :])
        if prune > 0 and d > 0 and C.shape[0] > 4:
            keep = rng.random(C.shape[0]) >= prune
            keep[:2] = True
            Cr = C.tocsr().tolil()
            for r in np.nonzero(~keep)[0]:
                Cr.rows[r] = []
                Cr.data[r] = []
            C = smat.csc_matrix(Cr.tocsr())
        out.append((smat.csc_matrix(W, dtype=np.float32), smat.csc_matrix(C, dtype=np.float32)))
    return out


def csr_with_empty_rows(X, rows):
    X = X.tolil()
    for r in rows:
        X.rows[r] = []
        X.data[r] = []
    X = X.tocsr().astype(np.float32)
    X.sort_indices()
    return X


HNSW_BUILD_SEED = 3


def save_hnsw_index(tmp, X, M, efC, metric, have_ref, threads=8):
    """Index of the rows X (dense float32, or scipy csr) trained by the reference library where oracle/_ref is built (returned,
    to search the saved file with), else built by this library's own index builder (pecos_b200/hnsw_build.py, same on-disk
    format; returns None).  The restatement the kernel is compared with bit for bit is pinned to the reference by
    tests/test_oracle_hnsw_cpu.py."""
    import json

    if not have_ref:
        from pecos_b200.hnsw_build import build_hnsw_index

        build_hnsw_index(X, tmp, M=M, efC=efC, metric=metric, seed=HNSW_BUILD_SEED)
        return None
    from oracle import ref

    r = ref.RefHNSW.train(X, M=M, efC=efC, metric=metric, threads=threads)
    os.makedirs(tmp, exist_ok=True)
    r.save(os.path.join(tmp, "c_model"))
    json.dump({"model": "HNSW", "data_type": r.data_type, "metric_type": metric, "num_item": int(X.shape[0]),
               "feat_dim": int(X.shape[1]), "pred_kwargs": {"efS": 50, "topk": 10, "threads": 1}},
              open(os.path.join(tmp, "param.json"), "w"))
    return r


def merge_shards_numpy(g_keys, g_ids, g_vals, g_cnt, k):
    """Reference semantics of the index-sharding merge (test-only): per query keep the k largest 64-bit keys
    among the valid entries of all ranks.  g_* have shape [world, rows, stride], g_cnt [world, rows]."""
    world, rows, stride = g_keys.shape
    out_ids = np.zeros((rows, k), dtype=np.uint32)
    out_vals = np.zeros((rows, k), dtype=np.float32)
    out_cnt = np.zeros(rows, dtype=np.uint32)
    for q in range(rows):
        cand = [(int(np.uint64(g_keys[g, q, r])), int(g_ids[g, q, r]), float(g_vals[g, q, r]))
                for g in range(world) for r in range(int(g_cnt[g, q]))]
        cand.sort(key=lambda t: -t[0])
        kk = min(k, len(cand))
        out_cnt[q] = kk
        for r in range(kk):
            out_ids[q, r], out_vals[q, r] = cand[r][1], cand[r][2]
    return out_ids, out_vals, out_cnt


def reachable_labels(layers):
    """Labels of the last layer with a complete path to the root (pruned trees drop rows of C at every layer).  The reference's
    predict_on_selected_outputs leaves the entry of an unreachable selected label UNINITIALISED and then indexes with it
    (pecos/core/xmc/inference.hpp:1302-1358), so in-contract selections only contain reachable labels."""
    reach = np.ones(1, dtype=bool)
    for _, C in layers:
        C = smat.csr_matrix(C)
        reach = np.asarray((C.astype(np.float32) @ reach.astype(np.float32)) > 0).ravel()
    return np.nonzero(reach)[0]


class RecordedReference(object):
    """Reference-library results that a test compares against, kept under tests/golden/ref_outputs/<name>.npz so that the
    comparison also runs where the reference library (oracle/_ref) is not built.

    With oracle/_ref present, `check` computes the reference result and compares in full (assert_csr_parity); with
    PB200_RECORD_REF_OUTPUTS=1 it also records it.  Without oracle/_ref it compares with the record: row sizes and label ids
    through a SHA-256 of the reference's (indptr, indices), scores at a fixed seeded sample of entries (`sample` per result)
    within the same relative tolerance.  The inputs of every recorded call are generated from fixed seeds by the test."""

    DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_outputs")

    def __init__(self, name, have_ref, sample=32):
        self.path = os.path.join(self.DIR, name + ".npz")
        self.live = bool(have_ref)
        self.record = self.live and os.environ.get("PB200_RECORD_REF_OUTPUTS") == "1"
        self.sample = sample
        self.store = {} if self.live else dict(np.load(self.path))
        self.used = set()

    @staticmethod
    def _pattern_digest(M):
        import hashlib

        h = hashlib.sha256()
        h.update(np.asarray(M.shape, dtype=np.int64).tobytes())
        h.update(np.asarray(M.indptr, dtype=np.int64).tobytes())
        h.update(np.asarray(M.indices, dtype=np.int64).tobytes())
        return np.frombuffer(h.digest(), dtype=np.uint8)

    def _positions(self, key, nnz):
        import zlib

        rng = np.random.default_rng(zlib.crc32(key.encode()))
        return np.sort(rng.choice(nnz, size=min(nnz, self.sample), replace=False)) if nnz else np.zeros(0, dtype=np.int64)

    def check(self, key, got, compute, rtol=1e-5, what=""):
        assert key not in self.used, f"duplicate key {key}"
        self.used.add(key)
        if self.live:
            want = compute()
            assert_csr_parity(got, want, rtol=rtol, what=what)
            if self.record:
                self.store[key + "|pattern"] = self._pattern_digest(want)
                self.store[key + "|values"] = np.asarray(want.data, dtype=np.float32)[self._positions(key, want.nnz)]
            return
        assert np.array_equal(self._pattern_digest(got), self.store[key + "|pattern"]), f"{what}: row sizes / label ids differ from the recorded reference"
        wd = self.store[key + "|values"]
        gd = np.asarray(got.data, dtype=np.float32)[self._positions(key, got.nnz)]
        rel = np.abs(gd.astype(np.float64) - wd.astype(np.float64)) / np.maximum(np.abs(wd), np.finfo(np.float32).tiny)
        assert rel.size == 0 or rel.max() <= rtol, f"{what}: max relative score error {rel.max():.3e} > {rtol} vs the recorded reference"

    def close(self):
        """Writes the record (recording runs only); a test must check every recorded result."""
        if self.record:
            os.makedirs(self.DIR, exist_ok=True)
            np.savez_compressed(self.path, **self.store)
        elif not self.live:
            assert {k.rsplit("|", 1)[0] for k in self.store} == self.used, "recorded reference results left unchecked"
