"""TEST INFRASTRUCTURE ONLY -- PairwiseANN checkers.

* :class:`RefPairwise` drives ``c_pairwise_ann_*`` of ``oracle/_ref/libpecos_float32.so`` (the unmodified reference library)
  with the prototypes of pecos/core/base.py:1966-2051.
* :func:`oracle_predict` runs the plain-C restatement of ``PairwiseANN::predict_single`` (``pairwise_oracle.c``) on in-memory
  X / Y_csc, or on a saved ``c_model`` folder through :func:`read_c_model`.
"""
import ctypes
import json
import os
from ctypes import POINTER, c_bool, c_char_p, c_float, c_int, c_uint32, c_uint64, c_void_p

import numpy as np
import scipy.sparse as smat

from pecos_b200.core import ScipyCscF32, ScipyCsrF32, ScipyDrmF32

from . import REF_LIB
from . import restatement

_ref = None


def ref_lib():
    global _ref
    if _ref is None:
        if not os.path.exists(REF_LIB):
            raise RuntimeError(f"{REF_LIB} missing: run `make -C oracle` where the reference sources are available")
        L = ctypes.CDLL(REF_LIB)
        for data_type, mat_t in (("drm", ScipyDrmF32), ("csr", ScipyCsrF32)):
            sfx = f"{data_type}_ip_f32"
            for name, res, args in (
                ("train", c_void_p, [POINTER(mat_t), POINTER(ScipyCscF32)]),
                ("load", c_void_p, [c_char_p, c_bool]),
                ("save", None, [c_void_p, c_char_p]),
                ("destruct", None, [c_void_p]),
                ("searchers_create", c_void_p, [c_void_p, c_uint32]),
                ("searchers_destruct", None, [c_void_p]),
                ("predict", None, [c_void_p, c_uint32, c_uint32, POINTER(mat_t), POINTER(c_uint32), POINTER(c_uint32),
                                   POINTER(c_uint32), POINTER(c_float), POINTER(c_float), c_bool]),
            ):
                f = getattr(L, f"c_pairwise_ann_{name}_{sfx}")
                f.restype, f.argtypes = res, args
        _ref = L
    return _ref


def _pymat(X):
    return (ScipyCsrF32.init_from(X), "csr") if isinstance(X, smat.csr_matrix) else (ScipyDrmF32.init_from(X), "drm")


class RefPairwise(object):
    """A reference PairwiseANN handle (train or load), its predict, save and destruct."""

    def __init__(self, ptr, data_type):
        self.ptr, self.data_type = c_void_p(ptr), data_type

    def _fn(self, name):
        return getattr(ref_lib(), f"c_pairwise_ann_{name}_{self.data_type}_ip_f32")

    @classmethod
    def train(cls, X, Y):
        pX, data_type = _pymat(X)
        pY = ScipyCscF32.init_from(smat.csc_matrix(Y, dtype=np.float32) if not isinstance(Y, smat.csc_matrix) else Y)
        return cls(getattr(ref_lib(), f"c_pairwise_ann_train_{data_type}_ip_f32")(pX, pY), data_type)

    @classmethod
    def load(cls, c_model_dir, data_type, lazy_load=False):
        return cls(getattr(ref_lib(), f"c_pairwise_ann_load_{data_type}_ip_f32")(c_model_dir.encode("utf-8"), lazy_load), data_type)

    def save(self, c_model_dir):
        self._fn("save")(self.ptr, str(c_model_dir).encode("utf-8"))

    def predict(self, Q, keys, topk, same=False, threads=1):
        """-> I, M, D, V of shape (len(keys), topk), zero-initialised like the reference's Python layer."""
        pQ, _ = _pymat(Q)
        keys = np.ascontiguousarray(keys, dtype=np.uint32)
        b = keys.shape[0]
        I = np.zeros(b * topk, np.uint32); M = np.zeros(b * topk, np.uint32)  # noqa: E702
        D = np.zeros(b * topk, np.float32); V = np.zeros(b * topk, np.float32)  # noqa: E702
        s = c_void_p(self._fn("searchers_create")(self.ptr, threads))
        try:
            self._fn("predict")(s, b, topk, pQ, keys.ctypes.data_as(POINTER(c_uint32)), I.ctypes.data_as(POINTER(c_uint32)),
                                M.ctypes.data_as(POINTER(c_uint32)), D.ctypes.data_as(POINTER(c_float)),
                                V.ctypes.data_as(POINTER(c_float)), same)
        finally:
            self._fn("searchers_destruct")(s)
        return tuple(a.reshape(b, topk) for a in (I, M, D, V))

    def __del__(self):
        if getattr(self, "ptr", None):
            self._fn("destruct")(self.ptr)
            self.ptr = None


def read_c_model(c_model_dir, data_type):
    """(X, Y_csc) stored in a saved c_model folder (pairwise.hpp:60-102, :206-243), in stored order."""
    blocks = iter(restatement.read_mmap_store(os.path.join(c_model_dir, "index.mmap_store")))
    u = lambda dt: np.ascontiguousarray(next(blocks)).view(dt)  # noqa: E731
    N, L, d = [int(u(np.uint32)[0]) for _ in range(3)]
    yr, yc, ynnz = int(u(np.uint32)[0]), int(u(np.uint32)[0]), int(u(np.uint64)[0])
    yptr, yidx, yval = u(np.uint64), u(np.uint32), u(np.float32)
    Y = smat.csc_matrix((yval, yidx.astype(np.int64), yptr.astype(np.int64)), shape=(yr, yc))
    Y.has_sorted_indices = False  # keep stored order: never let scipy sort it
    xr, xc, xnnz = int(u(np.uint32)[0]), int(u(np.uint32)[0]), int(u(np.uint64)[0])
    if data_type == "csr":
        xptr, xidx, xval = u(np.uint64), u(np.uint32), u(np.float32)
        X = smat.csr_matrix((xval, xidx.astype(np.int64), xptr.astype(np.int64)), shape=(xr, xc))
    else:
        X = u(np.float32).reshape(xr, xc)
    assert (N, L, d) == (yr, yc, xc) and xr == N and ynnz == Y.nnz
    return X, Y


def oracle_predict(X, Y_csc, Q, keys, topk, same=False, isa=0):
    """Restatement of c_pairwise_ann_predict_* -> I, M, D, V (len(keys), topk), zero-initialised.  Y_csc is used in stored
    order (indptr / indices / data as they are)."""
    L = restatement.lib()
    if not hasattr(L, "_pwo_ready"):
        L.pwo_predict.restype = c_int
        L.pwo_predict.argtypes = [c_int, c_int, c_uint32] + [c_void_p] * 3 + [c_uint32] + [c_void_p] * 6 + \
                                 [c_uint32, c_uint32, c_void_p, c_int] + [c_void_p] * 4
        L._pwo_ready = True
    sparse = isinstance(X, smat.csr_matrix)
    keep = []

    def arr(a, dt):
        a = np.ascontiguousarray(a, dtype=dt)
        keep.append(a)
        return a.ctypes.data

    keys = np.ascontiguousarray(keys, dtype=np.uint32)
    b = keys.shape[0]
    out = [np.zeros(b * topk, np.uint32), np.zeros(b * topk, np.uint32), np.zeros(b * topk, np.float32), np.zeros(b * topk, np.float32)]
    if sparse:
        xs = (arr(X.indptr, np.uint64), arr(X.indices, np.uint32), arr(X.data, np.float32))
        Qc = smat.csr_matrix(Q)
        qs = (arr(Qc.indptr, np.uint64), arr(Qc.indices, np.uint32), arr(Qc.data, np.float32))
    else:
        xs = (None, None, arr(X, np.float32))
        qs = (None, None, arr(Q, np.float32))
    rc = L.pwo_predict(1 if sparse else 0, isa, X.shape[1], *xs, Y_csc.shape[1], arr(Y_csc.indptr, np.uint64),
                       arr(Y_csc.indices, np.uint32), arr(Y_csc.data, np.float32), *qs, b, topk, keys.ctypes.data, 1 if same else 0,
                       *[o.ctypes.data for o in out])
    if rc != 0:
        raise ValueError("label key out of range")
    I, M, D, V = out
    return I.reshape(b, topk), M.reshape(b, topk), D.reshape(b, topk), V.reshape(b, topk)
