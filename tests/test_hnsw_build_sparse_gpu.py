"""GPU tests of the sparse (csr) HNSW builder: the distance kernels (csrc/hnsw_build_sparse.cu) against the restatement's
hno_sparse_distance BIT FOR BIT, and indices built on the GPU searched by the CUDA engine and the restatement (bit-identical ids
and distances) with a recall floor -- and, where oracle/_ref travelled, by the reference library on the same file."""
import os

import numpy as np
import pytest
import scipy.sparse as smat

from .test_hnsw_build_sparse_cpu import exact_topk, make_rows, recall, sparse_distance

pytestmark = pytest.mark.gpu


def random_rows(seed, n, D, nnz, long_rows=(), empty_every=0):
    """Rows with strictly ascending indices: half of each row's draws from a small hot set (so pairs share features), half
    uniform over [0, D); rows `long_rows` get 3000 draws (past every shared-memory chunk), every `empty_every`-th row none."""
    rng = np.random.default_rng(seed)
    indptr, idx, val = [0], [], []
    for i in range(n):
        k = 3000 if i in long_rows else int(rng.integers(0, 2 * nnz + 1))
        if empty_every and i % empty_every == 1:
            k = 0
        c = np.unique(np.concatenate([rng.integers(0, min(D, 96), k // 2), rng.integers(0, D, k - k // 2)])).astype(np.int32)
        idx.append(c)
        val.append(rng.standard_normal(c.size).astype(np.float32))
        indptr.append(indptr[-1] + c.size)
    return smat.csr_matrix((np.concatenate(val), np.concatenate(idx), np.array(indptr)), shape=(n, D), dtype=np.float32)


@pytest.mark.parametrize("D", [40, 100_000, 2_000_000])
@pytest.mark.parametrize("metric", ["ip", "l2"])
def test_distance_kernels_bit_exact(gpu_clib, D, metric):
    import torch

    from pecos_b200.hnsw_build import _SparseDevice

    n = 32_000 if D == 40 else 3000                  # D = 40: a block of 30,000 candidates (accumulators in global memory)
    X = random_rows(D + 1, n, D, 6 if D == 40 else 40, long_rows=(3, 17, 2500), empty_every=53)
    dev = torch.device("cuda", 0)
    sp = _SparseDevice(torch, X, metric, dev)
    rng = np.random.default_rng(D)
    # block kernel: a level made of a subset of the rows (positions != row ids), two candidate ranges
    ids_np = np.sort(rng.choice(n, size=n - 50, replace=False))
    ids_np = np.union1d(ids_np, [3, 17, 2500]).astype(np.int64)
    block = sp.block_for(torch.from_numpy(ids_np).to(dev))
    ranges = [(0, 200, 0, 900), (100, 400, 37, 1700)] + ([(0, 64, 1000, 31_000)] if D == 40 else [])
    for q0, q1, c0, c1 in ranges:
        out = block(q0, q1, c0, c1).cpu().numpy()
        assert out.shape == (q1 - q0, c1 - c0)
        qs = np.concatenate([rng.integers(q0, q1, 1500), np.flatnonzero(np.isin(ids_np[q0:q1], [3, 17, 2500, 1])) + q0])
        cs = rng.integers(c0, c1, qs.size)
        want = np.array([sparse_distance(X, ids_np[q], X, ids_np[c], metric) for q, c in zip(qs, cs)], dtype=np.float32)
        got = out[qs - q0, cs - c0]
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (q0, c0)
    # candidate-set kernel: width 512 with -1 padding, long and empty rows among the candidates
    T, C = 12, 512
    cand = rng.integers(0, n, (T, C)).astype(np.int64)
    cand[:, 5] = 3
    cand[:, 6] = 1                                    # an empty row
    cand[2, 7] = 2500
    for t in range(T):
        cand[t, C - 13 * t - 1:] = -1
    out = sp.cand_dist(torch.from_numpy(cand).to(dev)).cpu().numpy()
    torch.cuda.synchronize()
    ti = rng.integers(0, T, 3000)
    i, j = rng.integers(0, C, 3000), rng.integers(0, C, 3000)
    i[:40], j[:40] = 5, 7
    for t, a, b in zip(ti, i, j):
        if cand[t, a] < 0 or cand[t, b] < 0:
            assert np.isinf(out[t, a, b])
            continue
        want = sparse_distance(X, cand[t, a], X, cand[t, b], metric)
        assert out[t, a, b].view(np.uint32) == want.view(np.uint32), (t, a, b)
    work = sp.work.cpu().numpy()
    assert work[0] > 0 and work[1] > 0
    assert torch.cuda.current_device() == 0


# the shapes of test_hnsw_sparse_gpu.py::test_random_sparse_indices_match_reference_library; recall floor = recall@10 at
# efS = 200 of the reference-trained index (efC = 60, 8 threads) on the same rows and queries, minus 0.02, rounded down
# (measured on the CPU: 0.898, 0.910, 0.873, 0.921; the builder's CPU path reached 0.910, 0.922, 0.876, 0.926)
@pytest.mark.parametrize("N,D,nnz,M,metric,floor", [(5000, 30000, 80, 12, "ip", 0.87), (3000, 2000, 25, 8, "l2", 0.88),
                                                    (2000, 40, 4, 6, "ip", 0.85), (2500, 100000, 300, 16, "ip", 0.90)])
def test_gpu_built_sparse_index_search_parity_and_recall(tmp_path, gpu_clib, have_ref, N, D, nnz, M, metric, floor):
    from oracle import restatement
    from pecos_b200.hnsw import HNSW
    from pecos_b200.hnsw_build import build_hnsw_index

    X = make_rows(N + D, N, D, nnz, 61)
    Q = make_rows(N + D + 1, 300, D, nnz, 17, long_row=(11, min(D, 5000)))  # one row beyond the engine's shared-memory staging
    folder = str(tmp_path / "idx")
    stats = build_hnsw_index(X, folder, M=M, efC=60, metric=metric, seed=5, device="cuda:0")
    assert stats["block_postings"] > 0 and stats["candidate_entries"] > 0
    m = HNSW.load(folder)
    o = restatement.OracleHNSW(folder, isa=0)
    for efS, topk in [(10, 10), (64, 10), (200, 10), (5, 40), (600, 100)]:
        idx, dist = m.predict(Q, pred_params=HNSW.PredParams(efS=efS, topk=topk), ret_csr=False)
        oi, od = o.predict(Q, efS, topk)
        assert np.array_equal(idx, oi), f"ids vs restatement efS={efS} topk={topk}"
        assert np.array_equal(dist.view(np.uint32), od.view(np.uint32)), f"distance bits vs restatement efS={efS}"
    exact = exact_topk(Q, X, metric)
    gi, _ = m.predict(Q, pred_params=HNSW.PredParams(efS=200, topk=10), ret_csr=False)
    r = recall(gi, exact)
    assert r >= floor, r
    if have_ref:
        from oracle import ref

        rl = ref.RefHNSW.load(os.path.join(folder, "c_model"), metric, data_type="csr")
        ri, rd = rl.predict(Q, 200, 10, threads=8)
        assert np.array_equal(ri, gi) and np.array_equal(rd.view(np.uint32), o.predict(Q, 200, 10)[1].view(np.uint32))
        trained = ref.RefHNSW.train(X, M=M, efC=60, metric=metric, threads=8)
        ti, _ = trained.predict(Q, 200, 10, threads=8)
        assert r >= recall(ti, exact) - 0.02
