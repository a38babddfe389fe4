"""CPU test of the merged prefix layer (build_prefix_layer): layers 0 and 1 of a model as ONE one-chunk layer whose W is
[W0 | W1] (layer 1's columns in its column order) with a shared bias row -- the layout the prefix kernel's image is packed from."""
import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .util import random_tree


@pytest.mark.parametrize("sizes,bias", [([4, 64, 300], 1.0), ([8, 40, 200], 1.0), ([3, 7], -1.0)])
def test_prefix_layer_equals_numpy_merge(tmp_path, clib, sizes, bias):
    layers = random_tree(151, sizes, 300, 20, bias=bias)
    folder = str(tmp_path / "m")
    synth.save_xlinear_model(folder, layers, bias=bias, only_topk=5)
    got = clib.host_prefix_layer_layout(folder + "/ranker")
    W = smat.hstack([layers[0][0], layers[1][0]]).tocsc()
    want = clib.host_layer_layout_from_csc(W, smat.csc_matrix(np.ones((W.shape[1], 1), dtype=np.float32)), bias)[0]
    assert got["n_chunks"] == 1 and got["n_cols"] == sizes[0] + sizes[1] and got["w_rows"] == W.shape[0]
    for key in ("chunks", "meta", "entries"):
        assert np.array_equal(got[key], want[key]), key
    # and the entries rebuild the merged matrix exactly
    h = got["chunks"][0]
    R = int(h["nnz_rows"])
    rows = got["meta"][:R].astype(np.int64)
    rp = got["meta"][(R + 3) // 4 * 4:][: R + 1].astype(np.int64)
    dense = np.zeros(W.shape, dtype=np.float32)
    for r in range(R):
        e = got["entries"][rp[r]: rp[r + 1]]
        dense[rows[r], e["col_offset"].astype(np.int64)] += e["val"]
    assert np.array_equal(dense, W.toarray())
    assert int(h["has_bias"]) == (1 if bias > 0 and W[-1].nnz else 0)
