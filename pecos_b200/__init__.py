"""pecos_b200 -- H100-native (sm_90a) inference engine for PECOS's two retrieval hot paths.

* :class:`pecos_b200.xlinear.XLinearModel` -- XR-Linear beam-search prediction (``pecos.xmc.xlinear.XLinearModel`` API)
* :class:`pecos_b200.hnsw.HNSW` -- HNSW dense search (``pecos.ann.hnsw.HNSW`` API)

Both call hand-written CUDA kernels through the C ABI of ``pecos_b200/lib/libpecos_b200_float32.so``
(``include/pecos_b200.h``).  There is no CPU fallback.
"""
__version__ = "0.1.0"
