"""Multi-GPU XR-Linear prediction and HNSW search, one process per GPU (``torch.distributed``; NCCL on GPUs, gloo in CPU tests).

Two layouts for XR-Linear (SURVEY.md section 8e):

* **query sharding** -- model replicated, rows of ``X`` split across ranks; no data-path collective
  (:func:`split_rows_by_nnz`, used by ``bench.py`` and by callers that scatter their own batches).
* **index sharding** -- the leaf layer's weight chunks are split across ranks (:class:`ShardedXLinearModel`); the upper
  layers are replicated so every rank walks the same global beam, each rank scores only the leaf chunks it owns and keeps
  a local top-k as ``(key, label, score)`` with ``key = (orderable(score) << 32) | ~global_position``; ONE all-gather of
  those lists and a merge kernel give the global top-k, bit-identical to the single-GPU result.

HNSW index sharding (:class:`ShardedHNSW`): one independent graph per contiguous row range, each rank searches its own shard
and keeps its top-k as ``(key, global id, distance)`` with ``key = (~orderable(distance) << 32) | ~(rank * topk + slot)`` (one
fixed orderable for every NaN, after +inf); the same ONE all-gather and merge kernel give the top-k of the union, bit-identical
to merging the per-shard searches.

The reference has no inference-time model sharding (its parallelism is OpenMP threads inside one call,
pecos/core/xmc/inference.hpp:969-1005); this module is the multi-GPU counterpart of that loop.
"""
import dataclasses as dc
import json
import os
from ctypes import POINTER, byref, c_float, c_uint32, c_void_p

import numpy as np
import scipy.sparse as smat

from .core import ScipyCompressedSparseAllocator, ScipyCsrF32, XLINEAR_INFERENCE_MODEL_TYPES, get_clib

MERGE_CAPACITY = 1024  # world * stride records per query that the merge kernel holds (kSelKeys in csrc/shard_merge.cuh)


def split_rows_by_nnz(indptr, world):
    """Contiguous row blocks with (nearly) equal non-zeros: returns ``world + 1`` row boundaries."""
    indptr = np.asarray(indptr, dtype=np.int64)
    rows = indptr.size - 1
    total = int(indptr[-1])
    bounds = [0]
    for r in range(1, world):
        target = total * r // world
        b = int(np.searchsorted(indptr, target, side="left"))
        bounds.append(min(max(b, bounds[-1]), rows))
    bounds.append(rows)
    return bounds


class _TorchComm(object):
    """all_gather over torch.distributed for the fixed-shape local top-k buffers."""

    def __init__(self, group=None):
        import torch.distributed as dist

        self.dist = dist
        self.group = group
        self.rank = dist.get_rank(group)
        self.world = dist.get_world_size(group)

    def all_gather(self, local):
        import torch

        # concatenation along dim 0 is the layout both NCCL and gloo accept; rank r's block is out[r]
        shape = tuple(local.shape)
        out = torch.empty((self.world * shape[0],) + shape[1:], dtype=local.dtype, device=local.device)
        self.dist.all_gather_into_tensor(out, local.contiguous(), group=self.group)
        return out.view((self.world,) + shape)


class ShardedXLinearModel(object):
    """Leaf-layer index-sharded XR-Linear model: ``predict`` returns the same CSR matrix on every rank."""

    def __init__(self, c_model, rank, world, comm, clib, depth_params):
        self.model_chain = c_model
        self.rank, self.world = rank, world
        self.comm = comm
        self._clib = clib
        self.pred_params = depth_params

    def __del__(self):
        try:
            if self.model_chain is not None:
                self._clib.xlinear_destruct_model(self.model_chain)
                self.model_chain = None
        except Exception:
            pass

    @classmethod
    def load(cls, model_folder, comm=None, weight_matrix_type="BINARY_SEARCH_CHUNKED", device=None):
        clib = get_clib()
        clib.require_gpu()
        comm = comm or _TorchComm()
        if device is not None:
            clib.set_device(device)
        ranker = os.path.join(model_folder, "ranker")
        param = json.load(open(os.path.join(ranker, "param.json")))
        is_mmap = bool(param.get("is_mmap", False))
        type_id = -1 if is_mmap else XLINEAR_INFERENCE_MODEL_TYPES[weight_matrix_type]
        h = c_void_p(clib.clib_float32.pb200_xlinear_load_sharded(ranker.encode("utf-8"), type_id, comm.rank, comm.world))
        depth = int(param["depth"])
        pp = [json.load(open(os.path.join(ranker, f"{d}.model", "param.json")))["pred_kwargs"] for d in range(depth)]
        return cls(h, comm.rank, comm.world, comm, clib, pp)

    @property
    def shard(self):
        out = (c_uint32 * 4)()
        self._clib.clib_float32.pb200_xlinear_get_shard(self.model_chain, out)
        return tuple(int(x) for x in out)

    def predict(self, X, beam_size=None, only_topk=None, post_processor=None):
        """Every rank passes the same ``X`` (float32 CSR with sorted indices).  Raises ValueError before any GPU work when
        the queries are not such a matrix, the beam is too wide, or world x stride exceeds the merge capacity."""
        import torch

        if not isinstance(X, smat.csr_matrix):
            raise ValueError(f"type(X) = {type(X)} is not supported: index-sharded prediction takes csr queries only")
        if not X.has_sorted_indices:
            raise ValueError("Query matrix does not have sorted indices!")
        cx = ScipyCsrF32.init_from(X)  # refuses any dtype but float32, as XLinearModel.predict does
        self._clib.xlinear_check_plan(self.model_chain, beam_size, only_topk)
        k = int(only_topk or self.pred_params[-1]["only_topk"])
        # every rank sends `stride` records per query: k, or fewer where fewer candidates can exist at all
        stride = self._clib.xlinear_plan_stride(self.model_chain, beam_size, only_topk)
        if self.world * stride > MERGE_CAPACITY:
            narrow = f" (stride {stride} of top-k {k}: the most candidates a leaf row can hold)" if stride != k else ""
            raise ValueError(f"world * top-k = {self.world * stride}{narrow} exceeds the merge capacity of {MERGE_CAPACITY} "
                             f"records per query")
        c = self._clib.clib_float32
        rows = X.shape[0]
        dev = torch.device("cuda", c.pb200_get_device())
        # send buffer of the exchange: 16-byte {u64 key, u32 id, f32 value} records, viewed as int64 pairs for torch
        rec = torch.zeros((rows, stride, 2), dtype=torch.int64, device=dev)
        torch.cuda.synchronize(dev)
        pp = post_processor.encode("utf-8") if post_processor else None
        used = c.pb200_xlinear_sharded_local_csr_packed(self.model_chain, byref(cx), beam_size or 0, pp, only_topk or 0, stride,
                                                        rec.data_ptr())
        if used != stride:
            raise RuntimeError(f"pecos_b200: the engine used a stride of {used} records, the host plan {stride}")
        g_rec = self.comm.all_gather(rec)  # THE exchange: one all-gather of one buffer
        torch.cuda.synchronize(dev)
        self.last_exchange_bytes = int(rec.numel() * 8)
        alloc = ScipyCompressedSparseAllocator()
        c.pb200_xlinear_sharded_merge_packed(self.model_chain, self.world, rows, stride, only_topk or 0, g_rec.data_ptr(), alloc.cfunc)
        return alloc.get()


class ShardedHNSW(object):
    """HNSW index sharded by rows (``hnsw_build.build_hnsw_shards``): rank r searches only ``shard-<r>``; ``predict`` returns the
    same result on every rank.

    The result is NOT the search of one graph over all rows (each shard is its own graph: recall level against it); it is,
    bit for bit, the merge of the per-shard searches ordered by (distance with NaN last, shard rank, slot within the shard),
    with global ids ``row_begin[r] + local id``.  At world 1 this is the unsharded search when no NaN is returned; otherwise
    it is the unsharded search's entries ordered by (distance with NaN last, position): a NaN in the search heaps can leave
    the unsharded result out of order, and the merge sorts it."""

    MERGE_CAPACITY = MERGE_CAPACITY

    def __init__(self, index, manifest, rank, world, comm, clib):
        self.index = index
        self.manifest = manifest
        self.rank, self.world = rank, world
        self.comm = comm
        self._clib = clib
        self.row_begin = [int(b) for b in manifest["row_begin"]]
        self.num_item, self.feat_dim = int(manifest["num_item"]), int(manifest["feat_dim"])
        self.data_type, self.metric_type = manifest["data_type"], manifest["metric_type"]
        self.pred_params = index.PredParams.from_dict(manifest.get("pred_kwargs"))
        self.last_exchange_bytes = 0
        self.last_phase_ms = {}

    @classmethod
    def load(cls, folder, comm=None, device=None):
        from .hnsw import HNSW
        from .hnsw_build import SHARDS_MANIFEST

        with open(os.path.join(folder, SHARDS_MANIFEST), "r", encoding="utf-8") as f:
            manifest = json.load(f)
        comm = comm or _TorchComm()
        if int(manifest["world"]) != comm.world:
            raise ValueError(f"{folder} holds {manifest['world']} shards, the communicator has {comm.world} ranks")
        clib = get_clib()
        clib.require_gpu()
        if device is not None:
            clib.set_device(device)
        index = HNSW.load(os.path.join(folder, f"shard-{comm.rank}"))
        rb = manifest["row_begin"]
        if index.num_item != rb[comm.rank + 1] - rb[comm.rank] or index.feat_dim != manifest["feat_dim"]:
            raise ValueError(f"shard-{comm.rank} of {folder} does not match its manifest")
        return cls(index, manifest, comm.rank, comm.world, comm, clib)

    def get_pred_params(self):
        return dc.replace(self.pred_params)

    def predict(self, X, pred_params=None, ret_csr=True):
        """Every rank passes the same ``X``.  Same arguments and return types as ``HNSW.predict``: CSR (rows x num_item,
        distances as values) or ``(indices, distances)`` arrays rows x topk; slots beyond a row's results hold zeros."""
        import time

        import torch

        params = pred_params if pred_params is not None else self.get_pred_params()
        view, kind = self.index.create_pymat(X)
        if kind != self.data_type:
            raise ValueError(f"{kind} queries cannot be searched in a {self.data_type} index")
        if view.cols != self.feat_dim:
            raise ValueError(f"query dimension {view.cols} != index dimension {self.feat_dim}")
        n, k = int(view.rows), int(params.topk)
        if self.world * k > self.MERGE_CAPACITY:
            raise ValueError(f"world * topk = {self.world * k} exceeds the merge capacity of {self.MERGE_CAPACITY} records per query")
        if n and k:  # every shard has the manifest's width and the same M, so every rank decides alike, before the exchange
            self.index.check_search(params.efS, k)
        idx = np.zeros((n, k), dtype=np.uint32)
        dist = np.zeros((n, k), dtype=np.float32)
        if n and k:
            c = self._clib.clib_float32
            dev = torch.device("cuda", c.pb200_get_device())
            # send buffer of the exchange: 16-byte {u64 key, u32 id, f32 distance} records, viewed as int64 pairs for torch
            rec = torch.empty((n, k, 2), dtype=torch.int64, device=dev)
            torch.cuda.synchronize(dev)
            t0 = time.perf_counter()
            local = c.pb200_hnsw_sharded_local_packed_drm if kind == "drm" else c.pb200_hnsw_sharded_local_packed_csr
            local(self.index.model_ptr, byref(view), int(params.efS), k, self.rank, self.row_begin[self.rank], rec.data_ptr())
            t1 = time.perf_counter()
            g_rec = self.comm.all_gather(rec)  # THE exchange: one all-gather of one buffer
            torch.cuda.synchronize(dev)
            t2 = time.perf_counter()
            c.pb200_hnsw_sharded_merge_packed(self.index.model_ptr, self.world, n, k, g_rec.data_ptr(),
                                              idx.ctypes.data_as(POINTER(c_uint32)), dist.ctypes.data_as(POINTER(c_float)))
            t3 = time.perf_counter()
            self.last_exchange_bytes = int(rec.numel() * 8)
            self.last_phase_ms = {"local": 1e3 * (t1 - t0), "exchange": 1e3 * (t2 - t1), "merge": 1e3 * (t3 - t2)}
        if not ret_csr:
            return idx, dist
        row_starts = np.arange(n + 1, dtype=np.int64) * k
        return smat.csr_matrix((dist.ravel(), idx.ravel().astype(np.int64), row_starts), shape=(n, self.num_item), dtype=np.float32)
