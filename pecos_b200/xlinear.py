"""``XLinearModel`` -- predict-only mirror of ``pecos.xmc.xlinear.XLinearModel`` running on an H100.

Same names, argument meaning and error behaviour as the reference for the prediction path:

* ``XLinearModel.load(model_folder, is_predict_only=True, weight_matrix_type=...)``  pecos/xmc/xlinear/model.py:105-134
* ``XLinearModel.predict(X, pred_params=None, **kwargs)`` ........................... pecos/xmc/xlinear/model.py:480-550
* ``HierarchicalMLModel.load / predict`` (predict-only branch) ....................... pecos/xmc/base.py:1326-1369, :1577-1668
* ``PredParams.override_with_kwargs`` ............................................... pecos/xmc/base.py:1140-1173

* ``MLModel.load / predict`` (one layer of the python chain, ``is_predict_only=False``) .. pecos/xmc/base.py:832-878, :890-949

``predict_on_selected_outputs`` is served for predict-only handles and for the python chain (one
``c_xlinear_single_layer_predict_on_selected_outputs_*`` call per layer).  Training and pruning stay on the reference CPU library;
they are outside this engine's scope and raise ``NotImplementedError`` here.
"""
import copy
import dataclasses as dc
import json
from glob import glob
from os import path

import numpy as np
import scipy.sparse as smat

from .core import ScipyCompressedSparseAllocator, get_clib


@dc.dataclass
class MLModelPredParams(object):
    """Per-layer prediction parameters (pecos/xmc/base.py:652-682)."""

    only_topk: int = 20
    post_processor: str = "l3-hinge"

    @classmethod
    def from_layer_folder(cls, folder):
        param = json.loads(open(f"{folder}/param.json", "r", encoding="utf-8").read())
        kw = param.get("pred_kwargs", {}) or {}
        return cls(only_topk=int(kw.get("only_topk", 20)), post_processor=str(kw.get("post_processor", "l3-hinge")))


@dc.dataclass
class HierarchicalPredParams(object):
    """``HierarchicalMLModel.PredParams`` (pecos/xmc/base.py:1114-1173)."""

    model_chain: list = None

    def __len__(self):
        return len(self.model_chain)

    def override_with_kwargs(self, pred_kwargs):
        if pred_kwargs is None:
            return self
        if not isinstance(pred_kwargs, dict):
            raise TypeError("type(pred_kwargs) must be dict")
        overridden_beam_size = pred_kwargs.get("beam_size", None)
        overridden_only_topk = pred_kwargs.get("only_topk", None)
        overridden_post_processor = pred_kwargs.get("post_processor", None)
        depth = len(self.model_chain)
        for d in range(depth):
            if overridden_beam_size and d < (depth - 1):
                self.model_chain[d].only_topk = overridden_beam_size
            if overridden_only_topk and d == (depth - 1):
                self.model_chain[d].only_topk = overridden_only_topk
            if overridden_post_processor:
                self.model_chain[d].post_processor = overridden_post_processor
        return self


class MLModel(object):
    """One layer of the python prediction chain (pecos/xmc/base.py:598-949): holds ``W`` ((nr_features [+1]) x nr_labels,
    csc) and ``C`` (nr_labels x nr_codes, csc) on the host like the reference and predicts through
    ``c_xlinear_single_layer_predict_*``; the native side keeps the layer's chunked HBM layout in an LRU cache."""

    PredParams = MLModelPredParams

    def __init__(self, W, C=None, bias=-1.0, pred_params=None, **kwargs):
        if C is not None:
            if isinstance(C, smat.csr_matrix):
                C = C.tocsc()
            elif not isinstance(C, smat.csc_matrix):
                raise ValueError(f"type(C)={type(C)} is not supported")
        else:
            C = smat.csc_matrix(np.ones((W.shape[1], 1), dtype=W.dtype))  # pecos/xmc/base.py:632-634
        self.W = smat.csc_matrix(W, dtype=np.float32)
        self.W.sort_indices()
        self.C = smat.csc_matrix(C, dtype=np.float32)
        self.bias = float(bias)
        self.pred_params = self.PredParams() if pred_params is None else pred_params
        if self.C.shape[0] != self.W.shape[1]:
            raise ValueError("C.shape[0] != W.shape[1]")
        self._clib = get_clib()

    @property
    def nr_labels(self):
        return self.W.shape[1]

    @property
    def nr_codes(self):
        return self.C.shape[1]

    @property
    def nr_features(self):
        return self.W.shape[0] - (1 if self.bias > 0 else 0)

    @classmethod
    def load(cls, folder):
        """A ``<d>.model`` folder written by the reference's ``MLModel.save`` (param.json, W.npz, C.npz)."""
        param = json.loads(open(f"{folder}/param.json", "r", encoding="utf-8").read())
        assert param["model"] == "MLModel"
        W = smat.load_npz(f"{folder}/W.npz").tocsc().astype(np.float32)
        C = smat.load_npz(f"{folder}/C.npz").tocsc().astype(np.float32) if path.exists(f"{folder}/C.npz") else None
        return cls(W, C, float(param["bias"]), MLModelPredParams.from_layer_folder(folder))

    def get_pred_params(self):
        return copy.deepcopy(self.pred_params)

    def predict(self, X, csr_codes=None, pred_params=None, **kwargs):
        if X.shape[1] != self.nr_features:
            raise ValueError("Feature dimension of query matrix does not match weight matrix")
        pred_params = self.get_pred_params() if pred_params is None else copy.deepcopy(pred_params)
        if kwargs.get("only_topk", None):
            pred_params.only_topk = kwargs["only_topk"]
        if kwargs.get("post_processor", None):
            pred_params.post_processor = kwargs["post_processor"]
        if isinstance(X, smat.csr_matrix) and not X.has_sorted_indices:
            raise ValueError("Query matrix does not have sorted indices!")
        # the beam entering this layer: the widest row of the previous layer's prediction, or every parent
        if csr_codes is not None:
            b_prev = max(1, int(np.diff(smat.csr_matrix(csr_codes).indptr).max(initial=0)))
        else:
            b_prev = max(1, self.nr_codes)
        self._clib.xlinear_check_layer_beam(b_prev)
        pred_alloc = ScipyCompressedSparseAllocator()
        self._clib.xlinear_single_layer_predict(
            X,
            csr_codes,
            self.W,
            self.C,
            pred_params.post_processor,
            pred_params.only_topk if pred_params.only_topk else 0,
            kwargs.get("threads", -1),
            self.bias,
            pred_alloc,
        )
        return pred_alloc.get()


    def predict_on_selected_outputs(self, X, selected_outputs_csr, csr_codes=None, pred_params=None, **kwargs):
        """Scores of exactly the (instance, label) pairs of ``selected_outputs_csr`` for this layer (pecos/xmc/base.py:950-1012);
        ``csr_codes`` = the previous layer's selected-outputs result (must hold the parents of the selected labels)."""
        if X.shape[1] != self.nr_features:
            raise ValueError("Feature dimension of query matrix does not match weight matrix")
        if X.shape[0] != selected_outputs_csr.shape[0]:
            raise ValueError("Instance dimension of query and selected output matrix do not match")
        if selected_outputs_csr.shape[1] != self.nr_labels:
            raise ValueError("Label dimension of selected output matrix does not match")
        pred_params = self.get_pred_params() if pred_params is None else copy.deepcopy(pred_params)
        if kwargs.get("post_processor", None):
            pred_params.post_processor = kwargs["post_processor"]
        if isinstance(X, smat.csr_matrix) and not X.has_sorted_indices:
            raise ValueError("Query matrix does not have sorted indices!")
        pred_alloc = ScipyCompressedSparseAllocator()
        self._clib.xlinear_single_layer_predict_on_selected_outputs(
            X, selected_outputs_csr, csr_codes, self.W, self.C, pred_params.post_processor, kwargs.get("threads", -1), self.bias,
            pred_alloc)
        return pred_alloc.get()


class _PythonChain(object):
    """``HierarchicalMLModel`` with ``is_predict_only=False``: a list of ``MLModel`` (pecos/xmc/base.py:1669-1679)."""

    PredParams = HierarchicalPredParams

    def __init__(self, chain):
        self.model_chain = chain
        self.is_predict_only = False

    depth = property(lambda self: len(self.model_chain))
    nr_features = property(lambda self: self.model_chain[0].nr_features)
    nr_labels = property(lambda self: self.model_chain[-1].nr_labels)
    nr_codes = property(lambda self: self.model_chain[-1].nr_codes)

    def get_pred_params(self):
        return self.PredParams(model_chain=[m.get_pred_params() for m in self.model_chain])

    def predict(self, X, csr_codes=None, pred_params=None, **kwargs):
        assert X.dtype == np.float32
        if pred_params is None:
            pred_params = self.get_pred_params()
        else:
            pred_params = copy.deepcopy(pred_params)
        pred_params.override_with_kwargs(kwargs)
        pred_csr = csr_codes
        for d in range(self.depth):
            pred_csr = self.model_chain[d].predict(X, csr_codes=pred_csr, pred_params=pred_params.model_chain[d],
                                                   threads=kwargs.get("threads", -1))
        return pred_csr

    def predict_on_selected_outputs(self, X, selected_outputs_csr, csr_codes=None, pred_params=None, **kwargs):
        """Layer by layer (pecos/xmc/base.py:1772-1793): the selected set of layer d is the set of parents of layer d + 1's
        selection (pattern of ``selection @ C``); every layer scores exactly its selection with the previous result as codes."""
        assert X.dtype == np.float32
        if not isinstance(selected_outputs_csr, smat.csr_matrix):
            raise ValueError("type(selected_outputs_csr) = {} is not supported".format(type(selected_outputs_csr)))
        if selected_outputs_csr.shape[1] != self.nr_labels:
            raise ValueError("Label dimension of selected output matrix does not match")
        if X.shape[0] != selected_outputs_csr.shape[0]:
            raise ValueError("Instance dimension of query and selected output matrix do not match")
        pred_params = self.get_pred_params() if pred_params is None else copy.deepcopy(pred_params)
        pred_params.override_with_kwargs(kwargs)
        selections = [selected_outputs_csr.astype(np.float32)]
        for d in range(self.depth - 1, 0, -1):
            parents = (selections[0] @ self.model_chain[d].C).tocsr().astype(np.float32)
            parents.sort_indices()
            selections.insert(0, parents)
        pred_csr = csr_codes
        for d in range(self.depth):
            pred_csr = self.model_chain[d].predict_on_selected_outputs(X, selections[d], csr_codes=pred_csr,
                                                                       pred_params=pred_params.model_chain[d],
                                                                       threads=kwargs.get("threads", -1))
        return pred_csr


class HierarchicalMLModel(object):
    """Predict-only ``HierarchicalMLModel`` whose layers live in HBM behind an opaque C handle."""

    PredParams = HierarchicalPredParams

    def __init__(self, c_model, pred_params, clib):
        self.model_chain = c_model
        self.pred_params = pred_params
        self.is_predict_only = True
        self._clib = clib

    def __del__(self):
        try:
            if self.model_chain is not None:
                self._clib.xlinear_destruct_model(self.model_chain)
                self.model_chain = None
        except Exception:
            pass

    @property
    def depth(self):
        return self._clib.xlinear_get_int_attr(self.model_chain, "depth")

    @property
    def nr_features(self):
        return self._clib.xlinear_get_int_attr(self.model_chain, "nr_features")

    @property
    def nr_labels(self):
        return self._clib.xlinear_get_int_attr(self.model_chain, "nr_labels")

    @property
    def nr_codes(self):
        return self._clib.xlinear_get_int_attr(self.model_chain, "nr_codes")

    @property
    def weight_matrix_type(self):
        return self._clib.xlinear_get_layer_type(self.model_chain, 0)

    @classmethod
    def load(cls, model_folder, is_predict_only=True, **kwargs):
        clib = get_clib()
        param = json.loads(open(f"{model_folder}/param.json", "r", encoding="utf-8").read())
        assert param["model"] == "HierarchicalMLModel"
        depth = int(param.get("depth", len(glob("{}/*.model".format(model_folder)))))
        if not is_predict_only:
            if bool(param.get("is_mmap", False)):
                raise NotImplementedError("mmap single-layer handles (c_mlmodel_*) stay on the reference library")
            return _PythonChain([MLModel.load(f"{model_folder}/{d}.model") for d in range(depth)])
        is_mmap = bool(param.get("is_mmap", False))
        if is_mmap:
            model = clib.xlinear_load_mmap(model_folder, **kwargs)
        else:
            model = clib.xlinear_load_predict_only(model_folder, **kwargs)
        pred_params = cls.PredParams(
            model_chain=[MLModelPredParams.from_layer_folder(f"{model_folder}/{d}.model") for d in range(depth)]
        )
        return cls(model, pred_params, clib)

    def get_pred_params(self):
        return copy.deepcopy(self.pred_params)

    def _pred_chains(self, pred_params, kwargs):
        """(stored, requested) per-layer MLModelPredParams of a predict call."""
        if pred_params is None:
            pred_params = self.get_pred_params()
        elif isinstance(pred_params, self.PredParams):
            pred_params = copy.deepcopy(pred_params)
            if len(pred_params.model_chain) != self.depth:
                raise ValueError("len(pred_params.model_chain) != depth")
        else:
            raise ValueError("unknown type(pred_params)!!")
        pred_params.override_with_kwargs(kwargs)
        return self.get_pred_params().model_chain, pred_params.model_chain

    @staticmethod
    def _overridden_post_processor(old_chain, new_chain):
        """None if no layer's post_processor changed, else the one all layers now share (pecos/xmc/base.py:1630-1641)."""
        if all(o.post_processor == n.post_processor for (o, n) in zip(old_chain, new_chain)):
            return None
        if all(new_chain[0].post_processor == n.post_processor for n in new_chain):
            return new_chain[0].post_processor
        raise NotImplementedError("when is_predict_only=True, post_processor is not supported for overriddng")

    def predict(self, X, csr_codes=None, pred_params=None, **kwargs):
        assert X.dtype == np.float32
        assert isinstance(X, smat.csr_matrix) or (isinstance(X, np.ndarray) and X.flags["C_CONTIGUOUS"])
        assert X.shape[1] == self.nr_features
        old_chain, new_chain = self._pred_chains(pred_params, kwargs)
        if csr_codes is not None:
            raise NotImplementedError("is_predict_only=True did not support csr_codes being not None")

        # identical gating to pecos/xmc/base.py:1627-1654
        overridden_post_processor = self._overridden_post_processor(old_chain, new_chain)
        if all(o.only_topk == n.only_topk for (o, n) in zip(old_chain[:-1], new_chain[:-1])):
            overridden_beam_size = None
        elif all(new_chain[0].only_topk == n.only_topk for n in new_chain[:-1]):
            overridden_beam_size = new_chain[0].only_topk
        else:
            raise NotImplementedError("when is_predict_only=True, beam_size is not supported for overriding")

        # a beam too wide for the top-k kernels is a ValueError here, not a fatal error inside the predict call
        self._clib.xlinear_check_plan(self.model_chain, overridden_beam_size, new_chain[-1].only_topk)
        pred_alloc = ScipyCompressedSparseAllocator()
        self._clib.xlinear_predict(
            self.model_chain,
            X,
            overridden_beam_size,
            overridden_post_processor,
            new_chain[-1].only_topk,
            kwargs.get("threads", -1),
            pred_alloc,
        )
        return pred_alloc.get()


    def predict_on_selected_outputs(self, X, selected_outputs_csr, csr_codes=None, pred_params=None, **kwargs):
        """Scores of exactly the (instance, label) pairs of ``selected_outputs_csr`` (pecos/xmc/base.py:1670-1771).  Unlike the
        reference, which serves this from CSC-layout handles only, every pecos_b200 handle can."""
        if X.dtype != np.float32:
            raise ValueError("X.dtype = {} is not supported".format(X.dtype))
        if not isinstance(X, smat.csr_matrix) and not (isinstance(X, np.ndarray) and X.flags["C_CONTIGUOUS"]):
            raise ValueError("type(X) = {} is not supported".format(type(X)))
        if X.shape[1] != self.nr_features:
            raise ValueError("Feature dimension of query matrix does not match weight matrix")
        if not isinstance(selected_outputs_csr, smat.csr_matrix):
            raise ValueError("type(selected_outputs_csr) = {} is not supported".format(type(selected_outputs_csr)))
        if selected_outputs_csr.shape[1] != self.nr_labels:
            raise ValueError("Label dimension of selected output matrix does not match")
        if X.shape[0] != selected_outputs_csr.shape[0]:
            raise ValueError("Instance dimension of query and selected output matrix do not match")
        if csr_codes is not None:
            raise NotImplementedError("is_predict_only=True did not support csr_codes being not None")
        overridden_post_processor = self._overridden_post_processor(*self._pred_chains(pred_params, kwargs))
        pred_alloc = ScipyCompressedSparseAllocator()
        self._clib.xlinear_predict_on_selected_outputs(
            self.model_chain, X, selected_outputs_csr, overridden_post_processor, kwargs.get("threads", -1), pred_alloc
        )
        return pred_alloc.get()


class XLinearModel(object):
    """Predict-only ``XLinearModel`` (pecos/xmc/xlinear/model.py)."""

    @dc.dataclass
    class PredParams(object):
        hlm_args: HierarchicalPredParams = None

        def override_with_kwargs(self, pred_kwargs):
            self.hlm_args.override_with_kwargs(pred_kwargs)
            return self

    def __init__(self, model=None):
        self.model = model

    @property
    def depth(self):
        return self.model.depth

    @property
    def nr_features(self):
        return self.model.nr_features

    @property
    def nr_labels(self):
        return self.model.nr_labels

    @property
    def nr_codes(self):
        return self.model.nr_codes

    @property
    def is_predict_only(self):
        return self.model.is_predict_only

    @classmethod
    def load(cls, model_folder, is_predict_only=True, **kwargs):
        """kwargs: ``weight_matrix_type`` in {"BINARY_SEARCH_CHUNKED", "HASH_CHUNKED", "CSC"} (npz models),
        ``lazy_load`` (mmap models) -- same as the reference."""
        model = HierarchicalMLModel.load(path.join(model_folder, "ranker"), is_predict_only, **kwargs)
        return cls(model)

    def get_pred_params(self):
        return self.PredParams(hlm_args=self.model.get_pred_params())

    def predict(self, X, pred_params=None, selected_outputs_csr=None, **kwargs):
        if (pred_params is not None) and (not isinstance(pred_params, self.PredParams)):
            raise TypeError("type(pred_kwargs) is not supported")
        max_pred_chunk = kwargs.get("max_pred_chunk", 10**7)
        if max_pred_chunk is not None and not isinstance(max_pred_chunk, int):
            raise TypeError("type(max_pred_chunk) is not supported.")
        hlm_args = None if pred_params is None else pred_params.hlm_args
        if max_pred_chunk is None or max_pred_chunk >= X.shape[0]:
            if selected_outputs_csr is None:
                return self.model.predict(X, pred_params=hlm_args, **kwargs)
            return self.model.predict_on_selected_outputs(X, selected_outputs_csr, pred_params=hlm_args, **kwargs)
        Ys = []
        new_kwargs = kwargs.copy()
        new_kwargs.pop("max_pred_chunk", None)
        for i in range(0, X.shape[0], max_pred_chunk):
            sel = None if selected_outputs_csr is None else selected_outputs_csr[i : i + max_pred_chunk, :]
            Ys.append(self.predict(X[i : i + max_pred_chunk, :], pred_params=pred_params, selected_outputs_csr=sel, **new_kwargs))
        return smat.vstack(Ys, format="csr")

    @staticmethod
    def load_feature_matrix(src):
        """npz (sparse) or npy (dense) float32 features (pecos/xmc/xlinear/model.py, load_feature_matrix)."""
        if src.endswith(".npz"):
            return smat.load_npz(src).tocsr().astype(np.float32)
        return np.load(src).astype(np.float32)
