"""CPU tests of the sparse x sparse product: the restatement (tests/spmm_oracle.py) against the reference library and the
recorded goldens, the Python dispatch of B200CoreLib.sparse_matmul, its refusals, and the opt-in overlay."""
import ctypes
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as smat

from . import spmm_oracle as so

REFERENCE = os.environ.get("REFERENCE", "/root/reference")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = [(ez, si) for ez in (0, 1) for si in (0, 1)]


def test_goldens_reproduce_with_the_restatement():
    cases = so.load_goldens()
    assert {name for name, _ in cases} >= {"signed_zeros", "nan_inf", "dup_unsorted", "empty_rows", "zero_rows", "zero_cols"}
    for (name, fmt), (X, Y, exp) in cases.items():
        for flags in FLAGS:
            so.assert_same(so.restate(X, Y, *flags), exp[flags], f"{name}|{fmt}|{flags}")


def test_goldens_reproduce_with_the_reference(have_ref):
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    for (name, fmt), (X, Y, exp) in so.load_goldens().items():
        for flags in FLAGS:
            so.assert_same(so.reference(X, Y, *flags), exp[flags], f"{name}|{fmt}|{flags}")


@pytest.mark.parametrize("seed", range(12))
def test_restatement_equals_the_reference_on_random_cases(have_ref, seed):
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    rng = np.random.default_rng(seed)
    fmt = ("csr", "csc")[seed % 2]
    m, k, n = (int(v) for v in rng.integers(0, 12, 3))
    vals = lambda r, c: r.choice(np.array([-2, -1, -0.0, 0.0, 0.5, 1, 3, np.inf], dtype=np.float32), c)  # noqa: E731
    X = so.random_operand(rng, fmt, (m, k), 0.4, dup=0.3 * (seed % 3 == 0), shuffle=seed % 4 == 1, values=vals)
    Y = so.random_operand(rng, fmt, (k, n), 0.4, dup=0.3 * (seed % 5 == 0), shuffle=seed % 3 == 2, values=vals)
    for flags in FLAGS:
        so.assert_same(so.restate(X, Y, *flags), so.reference(X, Y, *flags), f"seed {seed} {flags}")


class _Stub:
    """Records the sparse-matmul calls a B200CoreLib makes; a GPU is 'visible', and pb200_spmm_fits answers `fits`."""

    def __init__(self, fits=1):
        self.calls, self.fits, self.fits_args = [], fits, []

    def pb200_device_count(self):
        return 1

    def pb200_spmm_fits(self, b_rows, b_nnz, out):
        self.fits_args.append((b_rows, b_nnz))
        return self.fits

    def _matmul(self, fmt):
        def f(pX, pY, alloc, ez, si, threads):
            self.calls.append((fmt, type(pX._obj).__name__, type(pY._obj).__name__, pX._obj.shape, pY._obj.shape, ez, si, threads))
        return f

    def __getattr__(self, name):
        if name.startswith("c_sparse_matmul_"):
            return self._matmul(name.split("_")[3])
        raise AttributeError(name)


def _stub_lib(fits=1):
    from pecos_b200.core import B200CoreLib

    lib = object.__new__(B200CoreLib)
    lib.clib_float32 = _Stub(fits)
    return lib


@pytest.mark.parametrize("xf,yf,x_heavier,want", [
    ("csr", "csr", False, ("csr", "ScipyCsrF32", "ScipyCsrF32")),
    ("csc", "csc", False, ("csc", "ScipyCscF32", "ScipyCscF32")),
    ("csc", "csr", True, ("csc", "ScipyCscF32", "ScipyCscF32")),   # Y.tocsc()
    ("csc", "csr", False, ("csr", "ScipyCsrF32", "ScipyCsrF32")),  # X.tocsr()
    ("csr", "csc", True, ("csr", "ScipyCsrF32", "ScipyCsrF32")),   # Y.tocsr()
    ("csr", "csc", False, ("csc", "ScipyCscF32", "ScipyCscF32")),  # X.tocsc()
])
def test_dispatch_matches_the_reference_branches(xf, yf, x_heavier, want):
    lib = _stub_lib()
    X = smat.random(20, 15, 0.5 if x_heavier else 0.1, format=xf, dtype=np.float32, random_state=1)
    Y = smat.random(15, 10, 0.1 if x_heavier else 0.5, format=yf, dtype=np.float32, random_state=2)
    try:
        lib.sparse_matmul(X, Y, eliminate_zeros=True, sorted_indices=False, threads=3)
    except Exception:  # the stub allocates nothing, so building the result fails after the call
        pass
    c = lib.clib_float32.calls
    assert len(c) == 1 and c[0][:3] == want and c[0][3:5] == ((20, 15), (15, 10)) and c[0][5:] == (True, False, 3)
    # the right operand of the traversal is what has to fit: csr Y's rows, csc X's columns
    b_rows, b_nnz = lib.clib_float32.fits_args[0]
    assert (b_rows, b_nnz) == ((15, Y.nnz) if want[0] == "csr" else (15, X.nnz))


def test_struct_inputs_dispatch_without_conversion():
    from pecos_b200.core import ScipyCsrF32

    lib = _stub_lib()
    X = ScipyCsrF32.init_from(smat.random(6, 5, 0.5, format="csr", dtype=np.float32, random_state=3))
    Y = ScipyCsrF32.init_from(smat.random(5, 4, 0.5, format="csr", dtype=np.float32, random_state=4))
    try:
        lib.sparse_matmul(X, Y)
    except Exception:
        pass
    assert lib.clib_float32.calls[0][:3] == ("csr", "ScipyCsrF32", "ScipyCsrF32")


def test_refusals_before_any_native_product(clib):
    lib = _stub_lib()
    with pytest.raises(ValueError, match="X.shape"):
        lib.sparse_matmul(smat.csr_matrix((3, 4), dtype=np.float32), smat.csr_matrix((5, 2), dtype=np.float32))
    assert lib.clib_float32.calls == [] and lib.clib_float32.fits_args == []
    # 2^40 entries never fit: the real library says so (with or without a device) and sparse_matmul raises MemoryError
    out = (ctypes.c_uint64 * 2)()
    assert clib.clib_float32.pb200_spmm_fits(1000, 1 << 40, out) == 0 and out[0] > (1 << 43)
    lib = _stub_lib(fits=0)
    with pytest.raises(MemoryError):
        lib.sparse_matmul(smat.random(4, 3, 0.5, format="csr", dtype=np.float32), smat.random(3, 2, 0.5, format="csr", dtype=np.float32))
    assert lib.clib_float32.calls == []


def test_no_gpu_means_runtime_error(clib):
    if clib.device_count() > 0:
        pytest.skip("a GPU is visible here")
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        clib.sparse_matmul(smat.random(4, 3, 0.5, format="csr", dtype=np.float32), smat.random(3, 2, 0.5, format="csr", dtype=np.float32))


def test_opt_in_overlay_on_the_reference_python_package(tmp_path, built, have_ref):
    if not os.path.isdir(os.path.join(REFERENCE, "pecos")):
        pytest.skip("the reference checkout is not on this box")
    if not have_ref:
        pytest.skip("oracle/_ref not built")
    scratch = str(tmp_path / "refpy")
    shutil.copytree(os.path.join(REFERENCE, "pecos"), os.path.join(scratch, "pecos"))
    subprocess.run(["chmod", "-R", "u+w", scratch], check=True)
    shutil.copy(os.path.join(ROOT, "oracle", "_ref", "libpecos_float32.so"), os.path.join(scratch, "pecos", "core", "libpecos_float32.so"))
    p = os.path.join(scratch, "pecos", "utils", "smat_util.py")
    src = open(p).read().replace("smat.sputils.get_index_dtype", "smat._sputils.get_index_dtype").replace("copy=False", "copy=None")
    open(p, "w").write(src)
    code = r"""
import sys, ctypes, json
sys.path.insert(0, %r); sys.path.insert(0, %r)
from pecos.core import clib
from pecos_b200 import integration
def where(fn):
    class I(ctypes.Structure):
        _fields_ = [("f", ctypes.c_char_p), ("b", ctypes.c_void_p), ("s", ctypes.c_char_p), ("a", ctypes.c_void_p)]
    dl = ctypes.CDLL(None); dl.dladdr.argtypes = [ctypes.c_void_p, ctypes.POINTER(I)]
    i = I(); dl.dladdr(ctypes.cast(fn, ctypes.c_void_p).value, ctypes.byref(i)); return i.f.decode()
names = ("c_sparse_matmul_csr_f32", "c_sparse_matmul_csc_f32")
out = {}
integration.overlay(clib, require_gpu=False)
out["default"] = [where(getattr(clib.clib_float32, n)) for n in names]
swapped = integration.overlay(clib, require_gpu=False, sparse_matmul=True)
out["opt_in"] = [where(getattr(clib.clib_float32, n)) for n in names]
out["swapped"] = [n for n in names if n in swapped]
out["argtypes"] = [len(getattr(clib.clib_float32, n).argtypes) for n in names]
print("RESULT" + json.dumps(out))
""" % (scratch, ROOT)
    r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
    import json

    out = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("RESULT")][0][6:])
    assert all(p.endswith("libpecos_float32.so") for p in out["default"]), out
    assert all(p.endswith("libpecos_b200_float32.so") for p in out["opt_in"]), out
    assert len(out["swapped"]) == 2 and out["argtypes"] == [6, 6]
