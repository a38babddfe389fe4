"""Overlay the GPU hot-path symbols onto a live ``pecos.core.clib`` (see INTEGRATION.md section 2).

``overlay(clib)`` re-points the XR-Linear predict-only and HNSW (dense and sparse) search function pointers of the reference's
``corelib`` instance (pecos/core/base.py:481-539, :1951-1964), and all seven PairwiseANN slots (base.py:1966-2051), at
``libpecos_b200_float32.so``; with ``sparse_matmul=True`` also ``c_sparse_matmul_{csr,csc}_f32`` (base.py:1461-1534).  Every other
symbol keeps using the reference CPU library.  The reference package itself is not imported here: pass its ``clib`` object in.
"""
import ctypes

from .core import LIB_PATH

XLINEAR_SYMBOLS = (
    "c_xlinear_load_model_from_disk",
    "c_xlinear_load_model_from_disk_ext",
    "c_xlinear_load_mmap_model_from_disk",
    "c_xlinear_compile_mmap_model",  # host-only writer of the reference's mmap format
    "c_xlinear_destruct_model",
    "c_xlinear_get_int_attr",
    "c_xlinear_get_layer_type",
    "c_xlinear_predict_csr_f32",
    "c_xlinear_predict_drm_f32",
    # predict_on_selected_outputs (the reference serves it from CSC handles; every pecos_b200 handle can)
    "c_xlinear_predict_on_selected_outputs_csr_f32",
    "c_xlinear_predict_on_selected_outputs_drm_f32",
    # python prediction chain (is_predict_only=False models): one layer per call, W / C handed over by the caller
    "c_xlinear_single_layer_predict_csr_f32",
    "c_xlinear_single_layer_predict_drm_f32",
    "c_xlinear_single_layer_predict_on_selected_outputs_csr_f32",
    "c_xlinear_single_layer_predict_on_selected_outputs_drm_f32",
    # single-layer mmap handles (load / attrs / predict / destruct swapped together: handles are library-specific)
    "c_mlmodel_compile_mmap_model",  # host-only writer
    "c_mlmodel_load_mmap_model",
    "c_mlmodel_destruct_model",
    "c_mlmodel_get_int_attr",
    "c_mlmodel_predict_csr_f32",
    "c_mlmodel_predict_drm_f32",
    "c_mlmodel_predict_on_selected_outputs_csr_f32",
    "c_mlmodel_predict_on_selected_outputs_drm_f32",
)
HNSW_SLOTS = ("load", "destruct", "searchers_create", "searchers_destruct", "predict", "save")
# PairwiseANN handles all come from one library (train is a deep copy and is served here), so every slot is swapped together
PAIRWISE_SLOTS = ("train", "load", "save", "destruct", "searchers_create", "searchers_destruct", "predict")
# opt-in: for small products (the python chain's `selected x C`) the host<->device copies can outweigh the CPU product
SPARSE_MATMUL_SYMBOLS = ("c_sparse_matmul_csr_f32", "c_sparse_matmul_csc_f32")


def overlay(clib, lib_path=LIB_PATH, require_gpu=True, sparse_matmul=False):
    """Returns the list of symbols that were re-pointed.  require_gpu=False only re-points (binding tests on a box without a
    GPU); any call into the re-pointed symbols then aborts with "no CUDA device visible" -- there is no CPU fallback.
    sparse_matmul=True also re-points the two sparse x sparse product symbols (off by default)."""
    b200 = ctypes.CDLL(lib_path)
    if require_gpu and b200.pb200_device_count() <= 0:
        raise RuntimeError("pecos_b200: no CUDA device visible and there is no CPU fallback")
    swapped = []
    for name in XLINEAR_SYMBOLS:
        ref = getattr(clib.clib_float32, name)
        fn = getattr(b200, name)
        fn.restype, fn.argtypes = ref.restype, ref.argtypes
        setattr(clib.clib_float32, name, fn)
        swapped.append(name)
    fn_dict = getattr(clib, "ann_hnsw_fn_dict", {})
    b200.pb200_hnsw_set_foreign.restype = None
    b200.pb200_hnsw_set_foreign.argtypes = [ctypes.c_int] + [ctypes.c_void_p] * 5
    for type_id, key in enumerate((("drm", "ip"), ("drm", "l2"), ("csr", "ip"), ("csr", "l2"))):
        data_type, metric = key
        if key not in fn_dict:
            continue
        # Indices trained by the reference are REFERENCE handles: hand the reference's own functions to the library, which
        # forwards every handle / searcher token it did not create itself (train stays on the reference).
        ref_fns = [fn_dict[key].get(slot) for slot in ("destruct", "searchers_create", "searchers_destruct", "predict", "save")]
        b200.pb200_hnsw_set_foreign(type_id, *[ctypes.cast(f, ctypes.c_void_p) if f is not None else None for f in ref_fns])
        for slot in HNSW_SLOTS:
            if slot not in fn_dict[key]:
                continue
            name = "c_ann_hnsw_{}_{}_{}_f32".format(slot, data_type, metric)
            ref = fn_dict[key][slot]
            fn = getattr(b200, name)
            fn.restype, fn.argtypes = ref.restype, ref.argtypes
            fn_dict[key][slot] = fn
            setattr(clib.clib_float32, name, fn)  # direct attribute users see the same function as fn_dict users
            swapped.append(name)
    pw_dict = getattr(clib, "pairwise_ann_fn_dict", {})
    for data_type in ("drm", "csr"):
        key = (data_type, "ip")
        if key not in pw_dict:
            continue
        for slot in PAIRWISE_SLOTS:
            name = "c_pairwise_ann_{}_{}_ip_f32".format(slot, data_type)
            ref = pw_dict[key][slot]
            fn = getattr(b200, name)
            fn.restype, fn.argtypes = ref.restype, ref.argtypes
            pw_dict[key][slot] = fn
            setattr(clib.clib_float32, name, fn)
            swapped.append(name)
    for name in SPARSE_MATMUL_SYMBOLS if sparse_matmul else ():
        ref = getattr(clib.clib_float32, name)
        fn = getattr(b200, name)
        fn.restype, fn.argtypes = ref.restype, ref.argtypes
        setattr(clib.clib_float32, name, fn)
        swapped.append(name)
    clib.clib_b200 = b200
    return swapped
