"""Sparse x sparse products at the kernels' tier limits (pecos_b200/csrc/spmm_engine.h), each on both sides, and through
several workspace tiles (PB200_SPMM_WORKSPACE_MB), including a row larger than one tile.  Every result is compared byte for
byte with the reference library (oracle/_ref) where it is built, else with the restatement (tests/spmm_oracle.py)."""
import numpy as np
import pytest

from . import spmm_oracle as so

pytestmark = pytest.mark.gpu

COUNT_WARP_MAX_PRODUCTS = 1024
FOLD_WARP_MAX_DISTINCT = 512
FOLD_WARP_MAX_PRODUCTS = 65536


def check(clib, have_ref, X, Y, what):
    infos = []
    for ez, si in ((0, 0), (0, 1), (1, 1)):
        got = so.call(clib.clib_float32, X, Y, ez, si)
        infos.append(clib.sparse_matmul_last_info())
        want = so.reference(X, Y, ez, si) if have_ref else so.restate(X, Y, ez, si)
        so.assert_same(got, want, f"{what} {ez}{si}")
    return infos[-1]


def one_row_over(rng, lens, width, dup_in_b=False):
    """X: one row with one entry per B row; Y: B rows of the given lengths over [0, width), shuffled (dup_in_b: every B row
    after the first repeats an index), values with cancellations."""
    ptr, idx = [0], []
    for k, L in enumerate(lens):
        row = list(rng.choice(width, size=L, replace=False))
        if dup_in_b and L > 1 and k > 0:
            row[-1] = row[0]
        idx.extend(row)
        ptr.append(len(idx))
    vals = rng.choice(np.array([-1.5, -1, -0.25, 0.25, 1, 3], dtype=np.float32), len(idx))
    Y = so.operand("csr", (len(lens), width), ptr, idx, vals)
    X = so.operand("csr", (1, len(lens)), [0, len(lens)], np.arange(len(lens)), rng.standard_normal(len(lens)))
    return X, Y


@pytest.mark.parametrize("products", [COUNT_WARP_MAX_PRODUCTS, COUNT_WARP_MAX_PRODUCTS + 1])
def test_symbolic_tier_by_products(gpu_clib, have_ref, products):
    rng = np.random.default_rng(products)
    # products spread over B rows of 100 entries on 400 indices: few distinct outputs, the count tier decides on products
    lens = [100] * (products // 100) + ([products % 100] if products % 100 else [])
    X, Y = one_row_over(rng, lens, 400)
    info = check(gpu_clib, have_ref, X, Y, f"products={products}")
    assert info["products"] == products
    assert (info["count_warp_rows"], info["count_cta_rows"]) == ((1, 0) if products <= COUNT_WARP_MAX_PRODUCTS else (0, 1))


@pytest.mark.parametrize("distinct", [FOLD_WARP_MAX_DISTINCT, FOLD_WARP_MAX_DISTINCT + 1])
@pytest.mark.parametrize("dup_in_b", [False, True])
def test_numeric_tier_by_distinct_outputs(gpu_clib, have_ref, distinct, dup_in_b):
    rng = np.random.default_rng(distinct)
    # the first B row touches every output index, the others a subset, some with a repeated index
    X, Y = one_row_over(rng, [distinct, 300, 200, 77], distinct, dup_in_b=dup_in_b)
    info = check(gpu_clib, have_ref, X, Y, f"distinct={distinct}")
    assert info["alloc_nnz"] == distinct
    assert (info["fold_warp_rows"], info["fold_cta_rows"]) == ((1, 0) if distinct <= FOLD_WARP_MAX_DISTINCT else (0, 1))


@pytest.mark.parametrize("extra", [0, 1])
def test_numeric_tier_by_products(gpu_clib, have_ref, extra):
    rng = np.random.default_rng(40 + extra)
    # 128 B rows of 512 entries over the same 512 indices: 65536 products, 512 distinct; one more entry tips it over
    lens = [512] * 128 + ([1] if extra else [])
    X, Y = one_row_over(rng, lens, 512, dup_in_b=False)
    info = check(gpu_clib, have_ref, X, Y, f"products={65536 + extra}")
    assert info["products"] == FOLD_WARP_MAX_PRODUCTS + extra and info["alloc_nnz"] == 512
    assert (info["fold_warp_rows"], info["fold_cta_rows"]) == ((1, 0) if extra == 0 else (0, 1))


def test_cta_tier_with_repeated_indices_in_b_rows(gpu_clib, have_ref):
    rng = np.random.default_rng(9)
    X, Y = one_row_over(rng, [3000, 700, 700, 5, 1200], 4000, dup_in_b=True)
    info = check(gpu_clib, have_ref, X, Y, "cta tier, non-canonical B")
    assert info["fold_cta_rows"] == 1 and info["count_cta_rows"] == 1


def test_several_tiles_and_a_row_larger_than_one_tile(gpu_clib, have_ref, monkeypatch):
    rng = np.random.default_rng(10)
    vals = lambda r, n: r.choice(np.array([-2, -1, 0.5, 1, 2], dtype=np.float32), n)  # noqa: E731
    X = so.random_operand(rng, "csr", (3000, 2000), 0.05, values=vals)
    Y = so.random_operand(rng, "csr", (2000, 1500), 0.05, values=vals)
    # about 3000 rows x (100 A entries + 1500 outputs) x 8 B: several MB, so a 1 MB budget needs many tiles
    monkeypatch.setenv("PB200_SPMM_WORKSPACE_MB", "1")
    many = check(gpu_clib, have_ref, X, Y, "1 MB workspace")
    monkeypatch.setenv("PB200_SPMM_WORKSPACE_MB", "4096")
    one = check(gpu_clib, have_ref, X, Y, "4 GB workspace")
    assert many["tiles"] > one["tiles"] + 4, (many, one)
    # a single row whose output and accumulator need more than the 1 MB budget: it runs as a tile of its own
    wide = so.operand("csr", (1, 60000), [0, 60000], np.arange(60000), np.ones(60000))
    diag = so.operand("csr", (60000, 60000), np.arange(60001), np.arange(60000), rng.standard_normal(60000))
    monkeypatch.setenv("PB200_SPMM_WORKSPACE_MB", "1")
    info = check(gpu_clib, have_ref, wide, diag, "row larger than a tile")
    assert info["alloc_nnz"] == 60000 and info["fold_cta_rows"] == 1
