"""Records tests/golden/spmm/cases.npz from the reference library (oracle/_ref): small sparse x sparse products through
c_sparse_matmul_{csr,csc}_f32 with threads=1, all four (eliminate_zeros, sorted_indices) combinations.

Cases: signed zeros, NaN / +-inf, NaN payloads, repeated and unsorted indices in both operands, empty rows / columns / matrices, and a random
product with cancellations.  Keys: "<case>|<fmt>|X|{shape,ptr,idx,val}", the same for Y, and
"<case>|<fmt>|<ez><si>|{indptr,indices,data,nnz}" (arrays up to indptr[-1]; nnz = the count handed to pred_alloc).

    python tests/golden/make_golden_spmm.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from tests import spmm_oracle as so  # noqa: E402

OUT = os.path.join(HERE, "spmm", "cases.npz")
INF, NAN = np.float32(np.inf), np.float32(np.nan)


def raw(fmt, shape, rows):
    """Operand from a list of major rows [(idx, val), ...] (rows of a csr, columns of a csc), taken as given."""
    ptr = np.cumsum([0] + [len(r) for r in rows])
    idx = [i for r in rows for i, _ in r]
    val = [v for r in rows for _, v in r]
    return so.operand(fmt, shape, ptr, idx, val)


def cases():
    out = {}
    # +0 starts every accumulator: an entry that only receives -0 products is +0; +0 + -0 = +0; x + (-x) = +0
    X = [[(0, -0.0), (1, 1.0)], [(1, -1.0), (2, 2.0)], [(0, 0.0)], [(2, -3.0)]]
    Y = [[(0, 1.0), (2, -1.0)], [(0, -0.0), (1, 0.5)], [(1, 0.25), (2, -0.0), (3, -1.0)]]
    out["signed_zeros"] = (X, Y, (4, 3), (3, 4))
    # inf * 0 = NaN, inf + (-inf) = NaN, overflow to inf, NaN stays through eliminate_zeros
    X = [[(0, INF), (1, 1.0)], [(0, 1e30), (1, -1e30)], [(1, NAN)], [(0, -INF), (1, INF)]]
    Y = [[(0, 1.0), (1, 0.0)], [(0, 1e30), (1, 2.0), (2, -0.0)]]
    out["nan_inf"] = (X, Y, (4, 2), (2, 3))
    # NaN payloads (signalling and quiet, both signs): which operand's payload a NaN product or sum carries
    sa, sb, qa = (np.array([u], dtype=np.uint32).view(np.float32)[0] for u in (0x7F800001, 0xFF800002, 0x7FC00003))
    X = [[(0, sa), (1, 1.0)], [(0, 1.0), (1, sb)], [(0, qa), (1, sa)], [(1, INF), (0, 0.0)]]
    Y = [[(0, sb), (1, 1.0), (2, qa)], [(0, 2.0), (1, sa), (2, -INF)]]
    out["nan_payloads"] = (X, Y, (4, 2), (2, 3))
    # repeated / unsorted indices in A rows and B rows; first touch differs from ascending order
    X = [[(2, 1.0), (0, 2.0), (2, -0.5)], [(1, 3.0), (1, 3.0)], [], [(0, 1.0), (1, 1.0), (2, 1.0)]]
    Y = [[(3, 1.0), (1, 2.0), (3, 4.0)], [(0, 1.0), (4, -1.0)], [(4, 1.5), (1, 0.5), (1, 0.5), (0, -2.0)]]
    out["dup_unsorted"] = (X, Y, (4, 3), (3, 5))
    # empty rows of X, rows of Y that are empty, a product without any entry, shapes with a zero
    X = [[], [(1, 1.0)], [], [(0, 2.0), (1, 0.0)]]
    Y = [[], [(0, 1.0), (2, 1.0)]]
    out["empty_rows"] = (X, Y, (4, 2), (2, 3))
    out["empty_product"] = ([[], [(1, 1.0)]], [[(0, 1.0)], []], (2, 2), (2, 1))
    out["zero_rows"] = ([], [[(0, 1.0)], []], (0, 2), (2, 1))
    out["zero_cols"] = ([[(0, 1.0)], [(1, 2.0)]], [[], []], (2, 2), (2, 0))
    out["zero_inner"] = ([[], []], [], (2, 0), (0, 3))
    return out


def as_format(fmt, rows, shape):
    """The case's lists as csr rows of `shape`, or as csc columns (the transposed matrix, shape reversed)."""
    return raw(fmt, shape if fmt == "csr" else (shape[1], shape[0]), rows)


def main():
    from oracle import have_ref

    if not have_ref():
        raise SystemExit("oracle/_ref is not built")
    store = {}
    specs = cases()
    rng = np.random.default_rng(20261018)
    for fmt in ("csr", "csc"):
        for name, (xr, yr, xs, ys) in specs.items():
            if fmt == "csr":
                X, Y = as_format(fmt, xr, xs), as_format(fmt, yr, ys)
            else:  # the columns of Y^T X^T are the rows of X Y: the csc traversal walks the same lists
                X, Y = as_format(fmt, yr, ys), as_format(fmt, xr, xs)
            store_case(store, name, fmt, X, Y)
        # random product with exact cancellations (values from a small set), repeated indices in both operands
        vals = lambda r, n: r.choice(np.array([-2, -1, -0.5, 0.5, 1, 2], dtype=np.float32), n)  # noqa: E731
        X = so.random_operand(rng, fmt, (40, 30), 0.2, dup=0.1, shuffle=True, values=vals)
        Y = so.random_operand(rng, fmt, (30, 50), 0.15, dup=0.1, shuffle=True, values=vals)
        store_case(store, "random", fmt, X, Y)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **store)
    print("wrote", OUT, len(store), "arrays")


def store_case(store, name, fmt, X, Y):
    assert X["shape"][1] == Y["shape"][0], (name, fmt, X["shape"], Y["shape"])
    for tag, op in (("X", X), ("Y", Y)):
        store[f"{name}|{fmt}|{tag}|shape"] = np.array(op["shape"], dtype=np.int64)
        for k in ("ptr", "idx", "val"):
            store[f"{name}|{fmt}|{tag}|{k}"] = op[k]
    for ez in (0, 1):
        for si in (0, 1):
            r = so.reference(X, Y, ez, si, threads=1)
            for k in ("indptr", "indices", "data"):
                store[f"{name}|{fmt}|{ez}{si}|{k}"] = r[k]
            store[f"{name}|{fmt}|{ez}{si}|nnz"] = np.array(r["nnz"], dtype=np.int64)


if __name__ == "__main__":
    main()
