"""Test infrastructure for the sparse x sparse product: raw compressed operands, the reference library's
c_sparse_matmul_{csr,csc}_f32 (oracle/_ref) driven through ctypes, and a NumPy restatement of the contract
(pecos/core/utils/matrix.hpp:1076-1290).

An operand is a dict {fmt, shape, ptr (u64), idx (u32), val (f32)} in csr or csc layout.  Its arrays are taken as they are, so
repeated and unsorted indices reach the library unchanged (scipy would canonicalise them).
"""
import ctypes
import os
from ctypes import POINTER, c_bool, c_int

import numpy as np

from pecos_b200.core import ScipyCompressedSparseAllocator, ScipyCscF32, ScipyCsrF32


def operand(fmt, shape, ptr, idx, val):
    return {"fmt": fmt, "shape": tuple(int(v) for v in shape), "ptr": np.ascontiguousarray(ptr, dtype=np.uint64),
            "idx": np.ascontiguousarray(idx, dtype=np.uint32), "val": np.ascontiguousarray(val, dtype=np.float32)}


def from_scipy(M):
    fmt = M.format
    assert fmt in ("csr", "csc")
    return operand(fmt, M.shape, M.indptr, M.indices, M.data)


def view(op):
    """ScipyCsrF32 / ScipyCscF32 over the operand's arrays (no copy)."""
    cls = ScipyCsrF32 if op["fmt"] == "csr" else ScipyCscF32
    v = cls()
    v.py_buf = op
    v.rows, v.cols = op["shape"]
    v.indptr = op["ptr"].ctypes.data_as(POINTER(ctypes.c_uint64))
    v.indices = op["idx"].ctypes.data_as(POINTER(ctypes.c_uint32))
    v.data = op["val"].ctypes.data_as(POINTER(ctypes.c_float))
    return v


class RawAllocator(ScipyCompressedSparseAllocator):
    """Keeps the nnz handed to pred_alloc and the raw arrays (the tail past indptr[-1] included)."""

    def __call__(self, is_col_major, rows, cols, nnz, indices_ptr, indptr_ptr, data_ptr):
        self.alloc_nnz = int(nnz)
        super().__call__(is_col_major, rows, cols, nnz, indices_ptr, indptr_ptr, data_ptr)

    def result(self):
        end = int(self.indptr[-1])
        return {"indptr": self.indptr.copy(), "indices": self.indices[:end].copy(), "data": self.data[:end].copy(),
                "nnz": self.alloc_nnz, "col_major": bool(self.is_col_major), "shape": (int(self.rows), int(self.cols))}


def bind(L):
    alloc = ScipyCompressedSparseAllocator.CFUNCTYPE
    L.c_sparse_matmul_csr_f32.restype = None
    L.c_sparse_matmul_csr_f32.argtypes = [POINTER(ScipyCsrF32), POINTER(ScipyCsrF32), alloc, c_bool, c_bool, c_int]
    L.c_sparse_matmul_csc_f32.restype = None
    L.c_sparse_matmul_csc_f32.argtypes = [POINTER(ScipyCscF32), POINTER(ScipyCscF32), alloc, c_bool, c_bool, c_int]
    return L


GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spmm", "cases.npz")
_ref = None


def ref_lib():
    global _ref
    if _ref is None:
        from oracle import REF_LIB

        _ref = bind(ctypes.CDLL(REF_LIB))
    return _ref


def call(L, X, Y, eliminate_zeros, sorted_indices, threads=1):
    """c_sparse_matmul_<fmt>_f32 of library L on two raw operands of one format; returns RawAllocator.result()."""
    assert X["fmt"] == Y["fmt"]
    alloc = RawAllocator()
    fn = getattr(L, "c_sparse_matmul_{}_f32".format(X["fmt"]))
    vx, vy = view(X), view(Y)
    fn(ctypes.byref(vx), ctypes.byref(vy), alloc.cfunc, bool(eliminate_zeros), bool(sorted_indices), threads)
    return alloc.result()


def reference(X, Y, eliminate_zeros, sorted_indices, threads=1):
    return call(ref_lib(), X, Y, eliminate_zeros, sorted_indices, threads)


def traversal(X, Y):
    """(A, B, n_out_rows): csr walks rows of X over rows of Y, csc columns of Y over columns of X."""
    if X["fmt"] == "csr":
        return X, Y, X["shape"][0]
    return Y, X, Y["shape"][1]


def restate(X, Y, eliminate_zeros, sorted_indices):
    """The contract in NumPy: per output row, acc_j = +0 then acc_j = acc_j + a_s * b_t (float32, separate roundings) over
    the traversal; indices ascending or in first-touch order; nnz before elimination; +-0 compacted out when asked."""
    A, B, n = traversal(X, Y)
    indptr = np.zeros(n + 1, dtype=np.uint64)
    indices, data = [], []
    nnz = 0
    with np.errstate(all="ignore"):
        for i in range(n):
            _restate_row(A, B, i, acc := {})
            nnz += len(acc)
            keys = sorted(acc) if sorted_indices else list(acc)
            for j in keys:
                if eliminate_zeros and acc[j] == 0:
                    continue
                indices.append(j)
                data.append(acc[j])
            indptr[i + 1] = len(indices)
    return {"indptr": indptr, "indices": np.array(indices, dtype=np.uint32), "data": np.array(data, dtype=np.float32),
            "nnz": nnz, "col_major": X["fmt"] == "csc", "shape": (X["shape"][0], Y["shape"][1])}


def _sse_nan(first, second):
    """The NaN x86 SSE returns: the first NaN operand made quiet, else (inf * 0, inf - inf) the default NaN 0xFFC00000."""
    for v in (first, second):
        if np.isnan(v):
            return np.array([np.float32(v).view(np.uint32) | 0x00400000], dtype=np.uint32).view(np.float32)[0]
    return np.array([0xFFC00000], dtype=np.uint32).view(np.float32)[0]


def _restate_row(A, B, i, acc):
    """Folds output row i into acc (insertion order = first touch).  A product's first SSE operand is the B value, a sum's
    the new product (the operand order of the reference's compiled loop; it only shows in NaN payloads)."""
    for s in range(int(A["ptr"][i]), int(A["ptr"][i + 1])):
        b, a = int(A["idx"][s]), A["val"][s]
        for t in range(int(B["ptr"][b]), int(B["ptr"][b + 1])):
            j, v = int(B["idx"][t]), B["val"][t]
            p = np.float32(a * v)
            if np.isnan(p):
                p = _sse_nan(v, a)
            old = acc.get(j, np.float32(0.0))
            r = np.float32(old + p)
            acc[j] = _sse_nan(p, old) if np.isnan(r) else r


def assert_same(got, want, what=""):
    """indptr, indices, data bits up to indptr[-1] and the allocator nnz byte-identical."""
    assert got["nnz"] == want["nnz"], f"{what}: allocator nnz {got['nnz']} != {want['nnz']}"
    assert got["col_major"] == want["col_major"] and tuple(got["shape"]) == tuple(want["shape"]), what
    assert np.array_equal(got["indptr"].astype(np.uint64), want["indptr"].astype(np.uint64)), f"{what}: indptr differs"
    assert np.array_equal(got["indices"].astype(np.uint32), want["indices"].astype(np.uint32)), f"{what}: indices differ"
    gd, wd = np.asarray(got["data"], dtype=np.float32), np.asarray(want["data"], dtype=np.float32)
    if not np.array_equal(gd.view(np.uint32), wd.view(np.uint32)):
        bad = np.nonzero(gd.view(np.uint32) != wd.view(np.uint32))[0]
        raise AssertionError(f"{what}: {bad.size} value bits differ; first at {bad[0]}: {gd[bad[0]]!r} != {wd[bad[0]]!r}")


# ------------------------------------------------------------------------------------------------------- operand builders
def random_operand(rng, fmt, shape, density, dup=0.0, shuffle=False, values=None):
    """Random operand of `shape`; dup: share of entries that repeat an earlier index of their row; shuffle: rows unsorted;
    values(rng, n): value generator (default normal)."""
    major, minor = (shape[0], shape[1]) if fmt == "csr" else (shape[1], shape[0])
    ptr, idx = [0], []
    for _ in range(major):
        k = rng.binomial(minor, density) if minor else 0
        row = list(np.sort(rng.choice(minor, size=k, replace=False))) if k else []
        if row and dup > 0:
            extra = [row[rng.integers(len(row))] for _ in range(rng.binomial(len(row), dup))]
            row = sorted(row + extra)
        if shuffle:
            rng.shuffle(row)
        idx.extend(row)
        ptr.append(len(idx))
    n = len(idx)
    val = values(rng, n) if values else rng.standard_normal(n)
    return operand(fmt, shape, ptr, idx, np.asarray(val, dtype=np.float32))


def transpose_layout(op):
    """The same matrix in the other layout (canonical operands only)."""
    import scipy.sparse as smat

    ctor = smat.csr_matrix if op["fmt"] == "csr" else smat.csc_matrix
    M = ctor((op["val"], op["idx"].astype(np.int64), op["ptr"].astype(np.int64)), shape=op["shape"])
    M = M.tocsc() if op["fmt"] == "csr" else M.tocsr()
    return from_scipy(M)


def load_goldens():
    """{(case, fmt): (X, Y, {(ez, si): expected})} from cases.npz."""
    E = np.load(GOLDEN)
    out = {}
    names = sorted({k.split("|")[0] + "|" + k.split("|")[1] for k in E.files})
    for nf in names:
        name, fmt = nf.split("|")
        ops = [operand(fmt, E[f"{nf}|{t}|shape"], E[f"{nf}|{t}|ptr"], E[f"{nf}|{t}|idx"], E[f"{nf}|{t}|val"]) for t in "XY"]
        exp = {}
        for ez in (0, 1):
            for si in (0, 1):
                p = f"{nf}|{ez}{si}|"
                exp[(ez, si)] = {"indptr": E[p + "indptr"], "indices": E[p + "indices"], "data": E[p + "data"],
                                 "nnz": int(E[p + "nnz"]), "col_major": fmt == "csc",
                                 "shape": (ops[0]["shape"][0], ops[1]["shape"][1])}
        out[(name, fmt)] = (ops[0], ops[1], exp)
    return out
