"""``PairwiseANN`` -- GPU counterpart of ``pecos.ann.pairwise.PairwiseANN`` (pecos/ann/pairwise/model.py).

For each (input, label) pair of a batch it returns the ``only_topk`` training inputs nearest to the input among the inputs
attached to the label (the rows of column ``label`` of ``Y``), with the reference's distances, order and ties, bit for bit.
The public surface is the reference's: ``TrainParams``, ``PredParams``, ``Searchers``, ``train``, ``load``, ``save``,
``searchers_create`` and ``predict``; folders saved by either library load in the other.  Only the inner-product metric
exists, as in the reference.  There is no CPU fallback: creating searchers or predicting without a visible CUDA device raises.
"""
import copy
import dataclasses as dc
import json
import os
from ctypes import POINTER, c_bool, c_char_p, c_float, c_uint32, c_void_p

import numpy as np
import scipy.sparse as smat

from .core import ScipyCscF32, ScipyCsrF32, ScipyDrmF32, get_clib


class _Params(object):
    _FULLNAME = None

    @classmethod
    def from_dict(cls, param=None):
        if param is None:
            return cls()
        if isinstance(param, cls):
            return copy.deepcopy(param)
        if isinstance(param, dict):
            return cls(**{f.name: copy.deepcopy(param[f.name]) for f in dc.fields(cls) if f.name in param})
        raise ValueError(f"{param} is not a valid parameter dictionary for {cls.__name__}")

    def to_dict(self, with_meta=True):
        d = {f.name: getattr(self, f.name) for f in dc.fields(self)}
        if with_meta:
            return dict({"__meta__": {"class_fullname": self._FULLNAME}}, **d)
        return d


class PairwiseANN(object):
    # class names the reference records in param.json (pecos.BaseClass.append_meta), so that saved folders are the same
    _FULLNAME = "pecos.ann.pairwise.model###PairwiseANN"

    @dc.dataclass
    class TrainParams(_Params):
        """metric_type: only "ip" (inner product) exists, as in the reference."""

        metric_type: str = "ip"
        _FULLNAME = "pecos.ann.pairwise.model###PairwiseANN.TrainParams"

    @dc.dataclass
    class PredParams(_Params):
        """batch_size: most (input, label) pairs per predict call; only_topk: neighbours returned per pair."""

        batch_size: int = 1024
        only_topk: int = 10
        _FULLNAME = "pecos.ann.pairwise.model###PairwiseANN.PredParams"

    class Searchers(object):
        """Native searcher token plus the result buffers of at most batch_size x only_topk slots."""

        def __init__(self, model, pred_params, num_searcher=1):
            self.searchers_ptr = None
            self.destruct_fn = model.fn_dict["searchers_destruct"]
            self.searchers_ptr = model.fn_dict["searchers_create"](model.model_ptr, num_searcher)
            self.pred_params = pred_params
            max_nnz = pred_params.batch_size * pred_params.only_topk
            self.Imat = np.zeros(max_nnz, dtype=np.uint32)
            self.Mmat = np.zeros(max_nnz, dtype=np.uint32)
            self.Dmat = np.zeros(max_nnz, dtype=np.float32)
            self.Vmat = np.zeros(max_nnz, dtype=np.float32)

        def __del__(self):
            if getattr(self, "searchers_ptr", None) is not None:
                self.destruct_fn(self.searchers_ptr)
                self.searchers_ptr = None

        def ctypes(self):
            return self.searchers_ptr

        def reset(self, reset_nnz):
            self.Imat[:reset_nnz].fill(0)
            self.Mmat[:reset_nnz].fill(0)
            self.Dmat[:reset_nnz].fill(0.0)
            self.Vmat[:reset_nnz].fill(0.0)

        def counters(self):
            """{pairs, distances, sparse_entries, replays} of the last predict call (replays: pairs whose ties were settled
            by replaying the reference's heap sequence)."""
            return get_clib().pairwise_ann_counters(self.searchers_ptr)

        def launch_info(self):
            """{stages, warps, per_warp_bytes, tiles} of the last predict call (see core.pairwise_ann_launch_info)."""
            return get_clib().pairwise_ann_launch_info(self.searchers_ptr)

    def __init__(self, model_ptr, num_input_keys, num_label_keys, feat_dim, fn_dict, pred_params=None):
        self.model_ptr = model_ptr
        self.num_input_keys = num_input_keys
        self.num_label_keys = num_label_keys
        self.feat_dim = feat_dim
        self.fn_dict = fn_dict
        self.pred_params = self.PredParams.from_dict(pred_params)

    def __del__(self):
        if getattr(self, "model_ptr", None):
            self.fn_dict["destruct"](self.model_ptr)
            self.model_ptr = None

    @property
    def data_type(self):
        return self.fn_dict["data_type"]

    @property
    def metric_type(self):
        return self.fn_dict["metric_type"]

    @staticmethod
    def create_pymat(X):
        if isinstance(X, (np.ndarray, ScipyDrmF32)):
            return (X if isinstance(X, ScipyDrmF32) else ScipyDrmF32.init_from(X)), "drm"
        if isinstance(X, (smat.csr_matrix, ScipyCsrF32)):
            return (X if isinstance(X, ScipyCsrF32) else ScipyCsrF32.init_from(X)), "csr"
        raise ValueError("type(X)={} is NOT supported!".format(type(X)))

    @classmethod
    def train(cls, X, Y, train_params=None, pred_params=None):
        """X: inputs (ndarray or csr_matrix, float32), Y: input-to-label matrix (csr or csc); both are copied."""
        train_params = cls.TrainParams.from_dict(train_params)
        pred_params = cls.PredParams.from_dict(pred_params)
        if not isinstance(Y, smat.csr_matrix) and not isinstance(Y, smat.csc_matrix):
            raise ValueError("type(Y) should be either a csr_matrix or csc_matrix.")
        pY = ScipyCscF32.init_from(Y.tocsc())
        pX, data_type = cls.create_pymat(X)
        if pX.rows != pY.rows:
            raise ValueError("X.shape[0]={} != Y.shape[0]={}".format(pX.rows, pY.rows))
        fn_dict = get_clib().pairwise_ann_init(data_type, train_params.metric_type)
        model_ptr = c_void_p(fn_dict["train"](pX, pY))
        return cls(model_ptr, pY.rows, pY.cols, pX.cols, fn_dict, pred_params)

    @classmethod
    def load(cls, model_folder, lazy_load=False):
        with open("{}/param.json".format(model_folder), "r") as fin:
            param = json.loads(fin.read())
        if param["model"] != cls.__name__:
            raise ValueError("param[model] != cls.__name__")
        if not ("data_type" in param and "metric_type" in param):
            raise ValueError("param.json did not have data_type or metric_type!")
        fn_dict = get_clib().pairwise_ann_init(param["data_type"], param["metric_type"])
        c_model_dir = f"{model_folder}/c_model"
        if not os.path.isdir(c_model_dir):
            raise ValueError(f"c_model_dir did not exist: {c_model_dir}")
        model_ptr = c_void_p(fn_dict["load"](c_char_p(c_model_dir.encode("utf-8")), c_bool(lazy_load)))
        pred_params = cls.PredParams.from_dict(param["pred_kwargs"])
        return cls(model_ptr, param["num_input_keys"], param["num_label_keys"], param["feat_dim"], fn_dict, pred_params)

    def save(self, model_folder):
        model_folder = str(model_folder)
        if not os.path.exists(model_folder):
            os.makedirs(model_folder)
        param = {
            "__meta__": {"class_fullname": self._FULLNAME},
            "model": self.__class__.__name__,
            "data_type": self.data_type,
            "metric_type": self.metric_type,
            "num_input_keys": self.num_input_keys,
            "num_label_keys": self.num_label_keys,
            "feat_dim": self.feat_dim,
            "pred_kwargs": self.pred_params.to_dict(),
        }
        with open("{}/param.json".format(model_folder), "w") as fout:
            fout.write(json.dumps(param, indent=True))
        c_model_dir = f"{model_folder}/c_model"
        self.fn_dict["save"](self.model_ptr, c_char_p(c_model_dir.encode("utf-8")))

    def get_pred_params(self):
        return copy.deepcopy(self.pred_params)

    def searchers_create(self, pred_params=None, num_searcher=1):
        if not self.model_ptr:
            raise ValueError("self.model_ptr must exist before using searchers_create()")
        if num_searcher <= 0:
            raise ValueError("num_searcher={} <= 0 is NOT valid".format(num_searcher))
        pred_params = self.get_pred_params() if pred_params is None else self.PredParams.from_dict(pred_params)
        self._check_searchable()
        return PairwiseANN.Searchers(self, pred_params, num_searcher)

    def _check_searchable(self):
        """Dense models wider than the engine's staging area can be trained and saved, not searched: ValueError here."""
        if self.data_type == "drm":
            get_clib().pairwise_ann_check_dense(self.feat_dim)

    def predict(self, input_feat, label_keys, searchers, is_same_input=False):
        """Returns Imat, Mmat, Dmat, Vmat, each (len(label_keys), only_topk): input ids, 1/0 presence mask, distances and Y
        values; pair b uses row (0 if is_same_input else b) of input_feat and column label_keys[b]."""
        input_feat_py, data_type = self.create_pymat(input_feat)
        if data_type != self.data_type:
            raise ValueError("data_type={} is NOT consistent with self.data_type={}".format(data_type, self.data_type))
        if input_feat_py.cols != self.feat_dim:
            raise ValueError("input_feat_py.cols={} is NOT consistent with self.feat_dim={}".format(input_feat_py.cols, self.feat_dim))
        if not isinstance(label_keys, np.ndarray):
            raise TypeError("type(label_keys) != np.array")
        if label_keys.ndim != 1:
            raise ValueError("label_keys must be one-dimensional")
        if not is_same_input and input_feat_py.rows != label_keys.shape[0]:
            raise ValueError("input_feat_py.rows != label_keys.shape[0]")
        if is_same_input and input_feat_py.rows < 1 and label_keys.shape[0] > 0:
            raise ValueError("is_same_input needs one input row")
        cur_bsz = label_keys.shape[0]
        if cur_bsz > searchers.pred_params.batch_size:
            raise ValueError("cur_batch_size > searchers.batch_size!")
        # the reference reads label keys unchecked (out of bounds); refused here before any native call
        if cur_bsz and (not np.issubdtype(label_keys.dtype, np.integer) or label_keys.min() < 0
                        or label_keys.max() >= self.num_label_keys):
            raise ValueError("label_keys must be integers in [0, num_label_keys={})".format(self.num_label_keys))
        self._check_searchable()
        keys = np.ascontiguousarray(label_keys, dtype=np.uint32)
        only_topk = searchers.pred_params.only_topk
        cur_nnz = cur_bsz * only_topk
        searchers.reset(cur_nnz)
        self.fn_dict["predict"](
            searchers.ctypes(),
            cur_bsz,
            only_topk,
            input_feat_py,
            keys.ctypes.data_as(POINTER(c_uint32)),
            searchers.Imat.ctypes.data_as(POINTER(c_uint32)),
            searchers.Mmat.ctypes.data_as(POINTER(c_uint32)),
            searchers.Dmat.ctypes.data_as(POINTER(c_float)),
            searchers.Vmat.ctypes.data_as(POINTER(c_float)),
            c_bool(is_same_input),
        )
        Imat = searchers.Imat[:cur_nnz].reshape(cur_bsz, only_topk)
        Mmat = searchers.Mmat[:cur_nnz].reshape(cur_bsz, only_topk)
        Dmat = searchers.Dmat[:cur_nnz].reshape(cur_bsz, only_topk)
        Vmat = searchers.Vmat[:cur_nnz].reshape(cur_bsz, only_topk)
        return Imat, Mmat, Dmat, Vmat
