"""ctypes binding of ``oracle/_ref/libsvsref_sq_build.so``: the reference's graph builder (``auto_build``) over
``SQDataset<int8_t / uint8_t>`` with a given scale and bias, and the distance that builder uses between two data,
compiled from the unmodified headers (``make -C oracle -f build_sq.mk build_sq``).
TEST INFRASTRUCTURE ONLY: the product package never imports it."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .bindings import HERE, METRIC_CODES, _c, _code, _ptr, effective_cpus


class RefSQBuildLib:
    """``svsref_sq_build`` / ``svsref_sq_build_distance``."""
    path = os.path.join(HERE, "_ref", "libsvsref_sq_build.so")

    def __init__(self, path: str | None = None):
        path = path or self.path
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.lib = C.CDLL(path)
        self.lib.svsref_sq_build_last_error.restype = C.c_char_p
        sz, vp, f = C.c_size_t, C.c_void_p, C.c_float
        self.lib.svsref_sq_build.argtypes = [C.c_int, vp, sz, sz, C.c_int, f, f, f, sz, sz, sz, sz, sz, vp, vp]
        self.lib.svsref_sq_build_distance.argtypes = [C.c_int, vp, sz, sz, C.c_int, f, f, vp, sz, vp]

    @classmethod
    def available(cls) -> bool:
        return os.path.exists(cls.path)

    def _check(self, rc):
        if rc:
            raise RuntimeError(self.lib.svsref_sq_build_last_error().decode())

    def build(self, codes: np.ndarray, scale: float, bias: float, metric: str, max_degree: int, window: int,
              alpha: float | None = None, max_candidates: int | None = None, prune_to: int | None = None,
              threads: int = 0):
        """Returns (graph uint32[n][R+1] degree-first, entry_point); the defaults as ``RefIntBuildLib.build``."""
        d = _c(codes)
        if d.dtype not in (np.int8, np.uint8):
            raise TypeError("int8 / uint8 codes only")
        n = d.shape[0]
        threads = threads or effective_cpus()
        if alpha is None:
            alpha = 1.2 if metric == "l2" else 0.95
        max_candidates = max_candidates or 3 * window
        prune_to = prune_to or (max_degree - 4 if max_degree >= 16 else max_degree)
        graph = np.zeros((n, max_degree + 1), dtype=np.uint32)
        ep = C.c_uint32()
        self._check(self.lib.svsref_sq_build(_code(d), _ptr(d), n, d.shape[1], METRIC_CODES[metric], scale, bias, alpha,
                                             max_degree, window, max_candidates, prune_to, threads, _ptr(graph),
                                             C.byref(ep)))
        return graph, int(ep.value)

    def distance(self, codes: np.ndarray, scale: float, bias: float, metric: str, pairs: np.ndarray) -> np.ndarray:
        """The builder's distance from datum i (its query) to datum j for every row (i, j) of ``pairs``: float32."""
        d = _c(codes)
        pr = np.ascontiguousarray(pairs, dtype=np.uint32).reshape(-1, 2)
        out = np.empty(pr.shape[0], dtype=np.float32)
        self._check(self.lib.svsref_sq_build_distance(_code(d), _ptr(d), d.shape[0], d.shape[1], METRIC_CODES[metric],
                                                      scale, bias, _ptr(pr), pr.shape[0], _ptr(out)))
        return out
