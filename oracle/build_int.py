"""ctypes binding of ``oracle/_ref/libsvsref_int.so``: the reference's graph builder (``auto_build``) over int8 /
uint8 rows, compiled from the unmodified headers (``make -C oracle -f build_int.mk build_int``).
TEST INFRASTRUCTURE ONLY: the product package never imports it."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .bindings import HERE, METRIC_CODES, _c, _code, _ptr, effective_cpus


class RefIntBuildLib:
    """``svsref_int_build``: the reference's ``auto_build`` over ``SimpleData<int8_t / uint8_t>``."""
    path = os.path.join(HERE, "_ref", "libsvsref_int.so")

    def __init__(self, path: str | None = None):
        path = path or self.path
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.lib = C.CDLL(path)
        self.lib.svsref_int_last_error.restype = C.c_char_p
        self.lib.svsref_int_build.argtypes = [C.c_int, C.c_void_p, C.c_size_t, C.c_size_t, C.c_int, C.c_float,
                                              C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p,
                                              C.c_void_p]

    @classmethod
    def available(cls) -> bool:
        return os.path.exists(cls.path)

    def build(self, data: np.ndarray, metric: str, max_degree: int, window: int, alpha: float | None = None,
              max_candidates: int | None = None, prune_to: int | None = None, threads: int = 0):
        """Returns (graph uint32[n][R+1] degree-first, entry_point); the defaults as ``RefLib.build``."""
        d = _c(data)
        if d.dtype not in (np.int8, np.uint8):
            raise TypeError("int8 / uint8 rows only")
        n = d.shape[0]
        threads = threads or effective_cpus()
        if alpha is None:
            alpha = 1.2 if metric == "l2" else 0.95
        # Defaults of index/vamana/index.h:1081-1095.
        max_candidates = max_candidates or 3 * window
        prune_to = prune_to or (max_degree - 4 if max_degree >= 16 else max_degree)
        graph = np.zeros((n, max_degree + 1), dtype=np.uint32)
        ep = C.c_uint32()
        rc = self.lib.svsref_int_build(_code(d), _ptr(d), n, d.shape[1], METRIC_CODES[metric], alpha, max_degree,
                                       window, max_candidates, prune_to, threads, _ptr(graph), C.byref(ep))
        if rc:
            raise RuntimeError(self.lib.svsref_int_last_error().decode())
        return graph, int(ep.value)
