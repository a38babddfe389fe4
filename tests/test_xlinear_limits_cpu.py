"""CPU checks behind tests/test_xlinear_limits_gpu.py: its model builders produce the quantities its cases claim to put on
each limit, its float64 reference agrees with the C restatement within its own bound, and the host-side beam check
accepts the widest beam the top-k kernels hold and rejects one more, as a ValueError from predict."""
import os

import numpy as np
import pytest
import scipy.sparse as smat

from pecos_b200 import synth

from .test_xlinear_limits_gpu import (CAP_D, CAP_WIDTHS, PFX_D, _cap_loop_layers, _cm_direct_fits, _dedup_first, _f64_check,
                                      _flat_layers, _prefix_budget_layers, _queries, _save, _two_layer)
from .util import random_tree

POST_PROCESSORS = ["noop", "sigmoid", "log-sigmoid", "l1-hinge", "l2-hinge", "l3-hinge", "l4-hinge", "l5-hinge",
                   "log-l1-hinge", "log-l3-hinge", "log-l4-hinge"]


def _host_layers(clib, folder):
    return clib.host_model_layout(os.path.join(folder, "ranker"))


def test_cover_model_has_exact_match_counts(tmp_path):
    """Every layer-1 chunk's rows are exactly features [0, R) and the bias row, so a query row with m features below R
    matches m rows of every chunk; widths 128 / 129 / 257 as built."""
    D, R = 2000, 600
    widths = [128, 129, 64, 257]
    layers = _two_layer(431, widths, D, 4, cover=R)
    W1, C1 = layers[1]
    assert W1.shape == (D + 1, sum(widths)) and C1.shape == (sum(widths), len(widths))
    c0 = 0
    for w in widths:
        rows = np.unique(smat.csc_matrix(W1)[:, c0:c0 + w].indices)
        assert np.array_equal(rows, np.r_[np.arange(R), D]), f"chunk of {w} columns covers other rows"
        c0 += w
    matches = [126, 127, 128, 129, 254, 255, 256, 257, 300, 300]
    nnz = [m + 40 for m in matches[:-2]] + [1024, 1025]
    X = _queries(441, D, nnz, cover=R, match_list=matches)
    got = np.diff(X.indptr)
    assert list(got[:10]) == nnz and got[10] == 0 and got[11] == nnz[0] and got[12] == 1025
    Xd = _dedup_first(X)
    assert np.diff(Xd.indptr)[12] == 1024  # the repeated index counts once
    per_row = np.asarray((Xd[:, :R] != 0).sum(axis=1)).ravel()
    assert list(per_row[:10]) == matches


def test_flat_and_two_layer_shapes_through_the_host_loader(tmp_path, clib):
    """The widths the limit cases rely on, read back as the engine reads them: widest chunk (c_max), W rows, chunk count;
    b_prev x c_max follows from them."""
    for width in (2048, 2049, 4096, 4097, 8064, 8065, 8192, 8193):
        folder = _save(str(tmp_path / f"flat{width}"), _flat_layers(1, width, 300, 4))
        (L,) = _host_layers(clib, folder)
        assert (L["n_chunks"], L["c_max"], L["w_rows"]) == (1, width, 301)
    for D in (16383, 16384):
        folder = _save(str(tmp_path / f"d{D}"), _two_layer(481, [8] * 16, D, 4))
        L0, L1 = _host_layers(clib, folder)
        assert L1["w_rows"] == D + 1 and L1["n_chunks"] == 16 and L1["c_max"] == 8 and L0["c_max"] == 16
    folder = _save(str(tmp_path / "qw"), _two_layer(401, [8] * 33, 1200, 4))
    L0, L1 = _host_layers(clib, folder)
    assert L0["c_max"] == 33 and L1["c_max"] == 8  # beam 32: 256 candidate floats; beam 33 > kQwSlots
    folder = _save(str(tmp_path / "wide_root"), _two_layer(451, [3] * 129, 800, 4))
    L0, L1 = _host_layers(clib, folder)
    assert L0["c_max"] == 129 and L1["n_chunks"] == 129 and L1["c_max"] == 3
    for widest in (256, 257):
        folder = _save(str(tmp_path / f"v{widest}"), _two_layer(491, [widest, 10, 100, 40], 500, 4))
        assert _host_layers(clib, folder)[1]["c_max"] == widest
    for n0, n1 in ((1, 50), (8, 248), (8, 249), (9, 60)):
        widths = synth._split_sizes(np.random.default_rng(511), n1, n0, even=True)
        folder = _save(str(tmp_path / f"p{n0}_{n1}"), _two_layer(512, list(widths), 600, 4))
        L0, L1 = _host_layers(clib, folder)
        assert L0["n_cols"] == n0 and L1["n_chunks"] == n0 and L0["n_cols"] + L1["n_cols"] == n0 + n1


@pytest.mark.parametrize("outside", [False, True])
def test_cap_loop_model_sits_on_the_edge(tmp_path, clib, outside):
    """The widest leaf chunk holds e entries (read back from the host layout), e fits an uncut 200-column image and e + 1
    does not; outside, the two 100-column ranges of the next cap (175) each fit."""
    layers, e = _cap_loop_layers(outside)
    assert _cm_direct_fits(CAP_D + 1, e - outside, 200) and not _cm_direct_fits(CAP_D + 1, e - outside + 1, 200)
    _, L1 = _host_layers(clib, _save(str(tmp_path / "m"), layers))
    ch = L1["chunks"]
    assert L1["c_max"] == 200 and L1["w_rows"] == CAP_D + 1 and list(ch["n_cols"]) == CAP_WIDTHS
    ent_end = np.r_[ch["ent_off"][1:], len(L1["entries"])]
    per_chunk = ent_end - ch["ent_off"]
    assert per_chunk.max() == per_chunk[0] == e
    offs = L1["entries"]["col_offset"][ch["ent_off"][0]:ent_end[0]]
    halves = np.bincount(np.minimum(offs // 100, 1), minlength=2)
    assert all(_cm_direct_fits(CAP_D + 1, int(h), 175) for h in halves)


@pytest.mark.parametrize("outside", [False, True])
def test_prefix_budget_model_sits_on_the_edge(tmp_path, clib, outside):
    """The merged prefix layer (host layout) has 64 columns, W rows 1001 and e entries; e fits next to 4 warps, e + 1 not."""
    layers, e = _prefix_budget_layers(outside)
    folder = _save(str(tmp_path / "m"), layers)
    M = clib.host_prefix_layer_layout(os.path.join(folder, "ranker"))
    assert (M["n_chunks"], M["c_max"], M["w_rows"], len(M["entries"])) == (1, 64, PFX_D + 1, e)
    assert _cm_direct_fits(PFX_D + 1, e - outside, 64) and not _cm_direct_fits(PFX_D + 1, e - outside + 1, 64)


@pytest.mark.parametrize("seed,sizes,beam,topk", [(61, [5], 0, 4), (62, [3, 20], 3, 6), (63, [4, 16, 90], 5, 7)])
def test_float64_reference_agrees_with_the_restatement(tmp_path, built, seed, sizes, beam, topk):
    """On small models and every post-processor, the restatement's scores (the reference's float32 arithmetic) sit within
    the float64 helper's bound, and for the flat model its top-k matches the float64 top-k up to that bound."""
    from oracle.restatement import OracleXLinear

    D = 120
    layers = random_tree(seed, sizes, D, 15, bias=1.0)
    folder = _save(str(tmp_path / "m"), layers)
    X = _queries(seed + 1, D, [20] * 12 + [40])
    o = OracleXLinear(os.path.join(folder, "ranker"))
    for pp in POST_PROCESSORS:
        got = o.predict(X, beam, pp, topk)
        assert got.nnz > 0
        _f64_check(layers, 1.0, X, got, pp, topk=topk if len(sizes) == 1 else None, what=f"restatement {sizes}")
        _f64_check(layers, 1.0, X.toarray(), o.predict(X.toarray(), beam, pp, topk), pp, what=f"restatement dense {sizes}")


def test_float64_reference_catches_a_wrong_score(tmp_path, built):
    """The bound is tight enough that one float32 ulp of headroom per layer is not a free pass: a score moved by 1e-4
    relative fails."""
    from oracle.restatement import OracleXLinear

    layers = random_tree(71, [4, 30], 100, 12, bias=1.0)
    folder = _save(str(tmp_path / "m"), layers)
    X = _queries(72, 100, [25] * 8)
    got = OracleXLinear(os.path.join(folder, "ranker")).predict(X, 4, "l3-hinge", 5)
    got.data[3] *= np.float32(1.0 + 1e-4)
    with pytest.raises(AssertionError, match="float64"):
        _f64_check(layers, 1.0, X, got, "l3-hinge")


@pytest.fixture(scope="module")
def wide_beam_folder(tmp_path_factory):
    layers = synth.make_tree_model(521, [16, 16000, 32000], 200, 4, bias=1.0)
    return _save(str(tmp_path_factory.mktemp("wide_beam")), layers)


def test_host_plan_check_at_the_beam_limit(wide_beam_folder, clib):
    """Layer 1 has 16 chunks of about 1,000 columns, so a beam of up to 16,000 can enter the leaf: 15,701 fits the block
    top-k, 15,702 does not; the widest fitting beam is reported either way."""
    c = clib.clib_float32
    h = c.pb200_xlinear_host_load(os.path.join(wide_beam_folder, "ranker").encode(), 0)
    try:
        assert clib.xlinear_check_plan(h, 15701, 10, host=True) == 15701
        assert clib.xlinear_check_plan(h, 1, 10, host=True) == 15701
        assert clib.xlinear_check_plan(h, 0, 0, host=True) == 15701  # stored only_topk (10)
        for beam in (15702, 16000, 1 << 31):
            with pytest.raises(ValueError, match="layer 2 would hold .* maximum of 15701; the widest beam_size that fits this model is 15701"):
                clib.xlinear_check_plan(h, beam, 10, host=True)
    finally:
        c.pb200_xlinear_host_free(h)
    # a model whose beams can never reach the limit fits every beam_size
    small = _save(os.path.join(wide_beam_folder, "small"), synth.make_tree_model(3, [4, 40], 50, 4, bias=1.0))
    h = c.pb200_xlinear_host_load(os.path.join(small, "ranker").encode(), 0)
    try:
        assert clib.xlinear_check_plan(h, 1 << 31, 10, host=True) is None
    finally:
        c.pb200_xlinear_host_free(h)


def test_predict_raises_value_error_before_any_gpu_work(wide_beam_folder, clib):
    """HierarchicalMLModel.predict runs the host check before the native predict call: the predict-only model below is
    backed by the host model alone, and its native predict must never be reached."""
    from pecos_b200.xlinear import HierarchicalMLModel, MLModelPredParams, XLinearModel

    c = clib.clib_float32
    h = c.pb200_xlinear_host_load(os.path.join(wide_beam_folder, "ranker").encode(), 0)

    class HostOnly(object):
        def xlinear_get_int_attr(self, model, attr):
            return {"depth": 3, "nr_features": 200}[attr]

        def xlinear_check_plan(self, model, beam, topk):
            return clib.xlinear_check_plan(model, beam, topk, host=True)

        def xlinear_predict(self, *args):
            raise AssertionError("the native predict call was reached")

        def xlinear_destruct_model(self, model):
            pass

    try:
        pp = HierarchicalMLModel.PredParams(model_chain=[MLModelPredParams(10, "l3-hinge") for _ in range(3)])
        m = XLinearModel(HierarchicalMLModel(h, pp, HostOnly()))
        X = _queries(1, 200, [10, 20])
        with pytest.raises(ValueError, match="15701"):
            m.predict(X, beam_size=15702, only_topk=10)
        with pytest.raises(AssertionError, match="native predict call was reached"):
            m.predict(X, beam_size=15701, only_topk=10)
    finally:
        c.pb200_xlinear_host_free(h)


def test_python_chain_layer_raises_value_error_before_the_native_call(clib, monkeypatch):
    """One layer of the is_predict_only=False chain (MLModel.predict) enters with a beam of max(row nnz of csr_codes) nodes,
    or every parent without codes.  Past 15,701 it raises ValueError before c_xlinear_single_layer_predict_* is called."""
    from pecos_b200.xlinear import MLModel

    def native(*args):
        raise AssertionError("the native single-layer call was reached")

    monkeypatch.setattr(clib, "xlinear_single_layer_predict", native)
    D, n = 10, 15702
    W = smat.csc_matrix(np.ones((D + 1, n), dtype=np.float32))
    X = _queries(2, D, [3, 4])
    for width in (15701, 15702):
        layer = MLModel(W, smat.identity(n, dtype=np.float32, format="csc"), bias=1.0)
        codes = smat.csr_matrix(np.ones((X.shape[0], n), dtype=np.float32)[:, :width], shape=(X.shape[0], width))
        codes.resize(X.shape[0], n)
        err = ValueError if width > 15701 else AssertionError
        with pytest.raises(err, match="15702 nodes" if width > 15701 else "native"):
            layer.predict(X, csr_codes=codes, only_topk=10)
    # without codes the beam is every parent: C.shape[1]
    for parents in (15701, 15702):
        layer = MLModel(W, smat.csc_matrix((np.ones(n, dtype=np.float32), (np.arange(n), np.arange(n) % parents)),
                                           shape=(n, parents)), bias=1.0)
        with pytest.raises(ValueError if parents > 15701 else AssertionError):
            layer.predict(X, only_topk=10)
