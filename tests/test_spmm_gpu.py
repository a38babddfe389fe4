"""Sparse x sparse products on the GPU (c_sparse_matmul_{csr,csc}_f32, B200CoreLib.sparse_matmul): byte-identical to the
reference's recorded goldens (tests/golden/make_golden_spmm.py) and to the live reference library (oracle/_ref)."""
import os
import threading

import numpy as np
import pytest
import scipy.sparse as smat

from . import spmm_oracle as so

pytestmark = pytest.mark.gpu
FLAGS = [(ez, si) for ez in (0, 1) for si in (0, 1)]


def gpu(clib, X, Y, ez, si):
    return so.call(clib.clib_float32, X, Y, ez, si)


def scipy_result(M):
    return {"indptr": M.indptr.astype(np.uint64), "indices": M.indices.astype(np.uint32), "data": M.data,
            "col_major": M.format == "csc", "shape": M.shape}


@pytest.mark.parametrize("fmt", ["csr", "csc"])
def test_goldens_both_entry_points_all_flags(gpu_clib, have_ref, fmt):
    cases = {k: v for k, v in so.load_goldens().items() if k[1] == fmt}
    assert len(cases) == 10
    for (name, _), (X, Y, exp) in cases.items():
        for flags in FLAGS:
            got = gpu(gpu_clib, X, Y, *flags)
            so.assert_same(got, exp[flags], f"{name}|{fmt}|{flags}")
            if have_ref:
                so.assert_same(got, so.reference(X, Y, *flags), f"{name}|{fmt}|{flags} vs oracle/_ref")


def _ref_dispatch(X, Y, ez, si):
    """The reference's four branches of corelib.sparse_matmul (base.py:1490-1532), on the reference library."""
    col = lambda M: isinstance(M, smat.csc_matrix)  # noqa: E731
    if col(X) and not col(Y):
        X, Y = (X, Y.tocsc()) if X.nnz > Y.nnz else (X.tocsr(), Y)
    elif not col(X) and col(Y):
        X, Y = (X, Y.tocsr()) if X.nnz > Y.nnz else (X.tocsc(), Y)
    r = so.reference(so.from_scipy(X), so.from_scipy(Y), ez, si, threads=1)
    return r


@pytest.mark.parametrize("xf,yf", [("csr", "csr"), ("csc", "csc"), ("csc", "csr"), ("csr", "csc")])
@pytest.mark.parametrize("x_heavier", [False, True])
def test_mixed_major_dispatch(gpu_clib, have_ref, xf, yf, x_heavier):
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    X = smat.random(60, 40, 0.3 if x_heavier else 0.05, format=xf, dtype=np.float32, random_state=1)
    Y = smat.random(40, 50, 0.05 if x_heavier else 0.3, format=yf, dtype=np.float32, random_state=2)
    for ez, si in FLAGS:
        Z = gpu_clib.sparse_matmul(X, Y, eliminate_zeros=bool(ez), sorted_indices=bool(si))
        want = _ref_dispatch(X, Y, ez, si)
        got = scipy_result(Z)
        got["nnz"] = gpu_clib.sparse_matmul_last_info()["alloc_nnz"]
        so.assert_same(got, want, f"{xf}x{yf} heavier={x_heavier} {ez}{si}")


def test_struct_inputs(gpu_clib):
    from pecos_b200.core import ScipyCscF32, ScipyCsrF32

    X = smat.random(30, 20, 0.3, format="csr", dtype=np.float32, random_state=3)
    Y = smat.random(20, 25, 0.3, format="csr", dtype=np.float32, random_state=4)
    want = gpu_clib.sparse_matmul(X, Y)
    got = gpu_clib.sparse_matmul(ScipyCsrF32.init_from(X), ScipyCsrF32.init_from(Y))
    assert got.format == "csr" and np.array_equal(got.indptr, want.indptr) and np.array_equal(got.indices, want.indices)
    assert np.array_equal(got.data.view(np.uint32), want.data.view(np.uint32))
    gc = gpu_clib.sparse_matmul(ScipyCscF32.init_from(X.tocsc()), ScipyCscF32.init_from(Y.tocsc()))
    assert gc.format == "csc" and np.allclose(gc.toarray(), (X @ Y).toarray(), rtol=1e-5, atol=1e-6)


def test_one_entry_with_100k_contributions_keeps_the_order(gpu_clib, have_ref):
    rng = np.random.default_rng(5)
    n = 100_000
    a = (rng.standard_normal(n) * np.float32(10.0) ** rng.integers(-6, 7, n)).astype(np.float32)
    b = np.ones(n, dtype=np.float32)
    # one A row of n entries, each over a one-entry B row on output index 0
    X = so.operand("csr", (1, n), [0, n], np.arange(n), a)
    Y = so.operand("csr", (n, 1), np.arange(n + 1), np.zeros(n), b)
    seq = np.float32(0.0)
    for v in a:
        seq = np.float32(seq + v)
    pairwise = np.float32(np.sum(a[::-1]))  # a re-associated sum
    assert pairwise.view(np.uint32) != seq.view(np.uint32), "the test values do not tell orders apart"
    got = gpu(gpu_clib, X, Y, 0, 1)
    assert got["data"].view(np.uint32)[0] == seq.view(np.uint32)
    if have_ref:
        so.assert_same(got, so.reference(X, Y, 0, 1), "100k contributions")


def zipf_pifa(seed, n, d, l, x_nnz_row, y_nnz_row):
    """Z = Y^T X: X (n x d) tf-idf-like rows, Y (n x l) label rows, Zipf feature and label frequencies; Y^T as csr."""
    rng = np.random.default_rng(seed)
    fp = 1.0 / np.arange(1, d + 1) ** 1.1
    lp = 1.0 / np.arange(1, l + 1) ** 1.2
    fp, lp = fp / fp.sum(), lp / lp.sum()

    def rows(m, width, k, p):
        ptr, idx = [0], []
        for _ in range(m):
            c = np.unique(rng.choice(width, size=max(1, rng.poisson(k)), p=p))
            idx.extend(c)
            ptr.append(len(idx))
        return smat.csr_matrix((rng.random(len(idx)).astype(np.float32) + 0.1, np.array(idx), np.array(ptr)), shape=(m, width))

    X = rows(n, d, x_nnz_row, fp)
    Y = rows(n, l, y_nnz_row, lp)
    return smat.csr_matrix(Y.T, dtype=np.float32), X.astype(np.float32)


def test_zipf_pifa_uses_every_tier(gpu_clib, have_ref):
    YT, X = zipf_pifa(7, 6000, 3000, 400, 40, 3)
    A, B = so.from_scipy(YT), so.from_scipy(X)
    for ez, si in FLAGS:
        got = gpu(gpu_clib, A, B, ez, si)
        info = gpu_clib.sparse_matmul_last_info()
        for k in ("count_warp_rows", "count_cta_rows", "fold_warp_rows", "fold_cta_rows"):
            assert info[k] > 0, (k, info)
        want = so.reference(A, B, ez, si, threads=os.cpu_count()) if have_ref else so.restate(A, B, ez, si)
        so.assert_same(got, want, f"pifa {ez}{si}")


def test_last_info_counts(gpu_clib):
    X = smat.random(50, 30, 0.2, format="csr", dtype=np.float32, random_state=8)
    Y = smat.random(30, 70, 0.2, format="csr", dtype=np.float32, random_state=9)
    Y.data[::3] = 0.0  # explicit zeros: kept as entries of Y, eliminated from Z where they cancel nothing else
    Z = gpu_clib.sparse_matmul(X, Y, eliminate_zeros=True)
    info = gpu_clib.sparse_matmul_last_info()
    blen = np.diff(Y.indptr)
    assert info["a_rows"] == 50
    assert info["products"] == int(sum(blen[X.indices]))
    S = smat.csr_matrix((np.ones_like(X.data), X.indices, X.indptr), shape=X.shape) @ \
        smat.csr_matrix((np.ones_like(Y.data), Y.indices, Y.indptr), shape=Y.shape)
    assert info["alloc_nnz"] == S.nnz
    assert info["kept_nnz"] == Z.nnz == int(np.count_nonzero(Z.data))
    assert info["tiles"] >= 2 and info["launches"] >= 3
    assert gpu_clib.clib_float32.pb200_spmm_last_kernel_ms() > 0.0


def test_two_threads_concurrently(gpu_clib):
    YT, X = zipf_pifa(11, 3000, 2000, 300, 30, 3)
    A, B = so.from_scipy(YT), so.from_scipy(X)
    want = {si: gpu(gpu_clib, A, B, 0, si) for si in (0, 1)}
    errors = []

    def work(si):
        try:
            for _ in range(3):
                so.assert_same(gpu(gpu_clib, A, B, 0, si), want[si], f"thread si={si}")
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    th = [threading.Thread(target=work, args=(si,)) for si in (0, 1)]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors


def test_opt_in_overlay_on_a_reference_corelib(gpu_clib, have_ref):
    """overlay(..., sparse_matmul=True) on a stand-in corelib over oracle/_ref re-points both symbols, and the reference's own
    call sequence through them gives the reference's bytes; the default overlay leaves them alone."""
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    import ctypes

    from oracle import REF_LIB
    from oracle import ref as oref
    from pecos_b200 import integration

    class StandIn:
        pass

    for opt_in in (False, True):
        c = StandIn()
        c.clib_float32 = so.bind(oref.bind(ctypes.CDLL(REF_LIB)))
        names = integration.overlay(c, sparse_matmul=opt_in)
        assert (set(integration.SPARSE_MATMUL_SYMBOLS) <= set(names)) == opt_in
        X = so.from_scipy(smat.random(40, 30, 0.2, format="csr", dtype=np.float32, random_state=12))
        Y = so.from_scipy(smat.random(30, 20, 0.2, format="csr", dtype=np.float32, random_state=13))
        got = so.call(c.clib_float32, X, Y, 1, 1)
        so.assert_same(got, so.reference(X, Y, 1, 1), "overlay")
