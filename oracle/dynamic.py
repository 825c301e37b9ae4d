"""ctypes binding of ``oracle/_ref/libsvsref_dynamic.so``: the reference's ``MutableVamanaIndex``
(index/vamana/dynamic_index.h) compiled from the unmodified headers (``make -C oracle -f dynamic.mk dynamic``).
TEST INFRASTRUCTURE ONLY: the product package never imports it."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .bindings import HERE, METRIC_CODES, _c, _code, _ptr, effective_cpus


class RefDynamic:
    """The reference's ``MutableVamanaIndex`` (index/vamana/dynamic_index.h) behind ``svsref_dynamic_*``."""

    def __init__(self, lib, handle, dtype, max_degree):
        self._lib, self._h, self._dtype, self.max_degree = lib, handle, np.dtype(dtype), max_degree

    def close(self):
        if self._h:
            self._lib.svsref_dynamic_destroy(self._h)
            self._h = None

    __del__ = close

    def _check(self, rc):
        if rc:
            raise RuntimeError(self._lib.svsref_dynamic_last_error().decode())

    def set_params(self, alpha, window, max_candidates, prune_to):
        self._check(self._lib.svsref_dynamic_set_params(self._h, float(alpha), window, max_candidates, prune_to))

    def add(self, points, ids, reuse_empty=False) -> np.ndarray:
        pts = _c(np.asarray(points).astype(self._dtype, copy=False))
        ids = _c(np.asarray(ids, dtype=np.uint64))
        slots = np.empty(len(ids), dtype=np.uint64)
        self._check(self._lib.svsref_dynamic_add(self._h, _ptr(pts), len(ids), _ptr(ids), int(reuse_empty), _ptr(slots)))
        return slots

    def delete(self, ids):
        ids = _c(np.atleast_1d(np.asarray(ids, dtype=np.uint64)))
        self._check(self._lib.svsref_dynamic_delete(self._h, _ptr(ids), len(ids)))

    def consolidate(self):
        self._check(self._lib.svsref_dynamic_consolidate(self._h))

    def compact(self):
        self._check(self._lib.svsref_dynamic_compact(self._h))

    def export(self):
        """(graph uint32[slots][R+1] degree first, status uint8 (0 Empty, 1 Valid, 2 Deleted), external ids
        (2^64 - 1 where not Valid), entry point) over every slot."""
        n = self._lib.svsref_dynamic_slots(self._h)
        graph = np.zeros((n, self.max_degree + 1), dtype=np.uint32)
        status = np.zeros(n, dtype=np.uint8)
        ext = np.zeros(n, dtype=np.uint64)
        ep = C.c_uint32()
        self._check(self._lib.svsref_dynamic_export(self._h, _ptr(graph), _ptr(status), _ptr(ext), C.byref(ep)))
        return graph, status, ext, int(ep.value)

    def search(self, queries, k, window, capacity=None):
        q = _c(np.asarray(queries, dtype=np.float32))
        capacity = window if capacity is None else capacity
        ids = np.empty((q.shape[0], k), dtype=np.uint64)
        dists = np.empty((q.shape[0], k), dtype=np.float32)
        self._check(self._lib.svsref_dynamic_search(self._h, _ptr(q), q.shape[0], k, window, capacity, _ptr(ids),
                                                    _ptr(dists)))
        return ids, dists


class RefDynamicLib:
    """The compiled façade (``oracle/_ref/libsvsref_dynamic.so``)."""
    path = os.path.join(HERE, "_ref", "libsvsref_dynamic.so")

    @classmethod
    def available(cls) -> bool:
        return os.path.exists(cls.path)

    def __init__(self, path=None):
        path = path or self.path
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.lib = L = C.CDLL(path)
        sz, vp = C.c_size_t, C.c_void_p
        L.svsref_dynamic_last_error.restype = C.c_char_p
        L.svsref_dynamic_create.restype = vp
        L.svsref_dynamic_create.argtypes = [C.c_int, vp, sz, sz, vp, sz, C.c_uint32, C.c_int, vp, C.c_float, sz, sz, sz, sz]
        L.svsref_dynamic_build.restype = vp
        L.svsref_dynamic_build.argtypes = [C.c_int, vp, sz, sz, C.c_int, C.c_float, sz, sz, sz, sz, vp, sz]
        L.svsref_dynamic_destroy.argtypes = [vp]
        L.svsref_dynamic_set_params.argtypes = [vp, C.c_float, sz, sz, sz]
        L.svsref_dynamic_add.argtypes = [vp, vp, sz, vp, C.c_int, vp]
        L.svsref_dynamic_delete.argtypes = [vp, vp, sz]
        L.svsref_dynamic_consolidate.argtypes = [vp]
        L.svsref_dynamic_compact.argtypes = [vp]
        L.svsref_dynamic_slots.restype, L.svsref_dynamic_slots.argtypes = sz, [vp]
        L.svsref_dynamic_export.argtypes = [vp, vp, vp, vp, C.POINTER(C.c_uint32)]
        L.svsref_dynamic_search.argtypes = [vp, vp, sz, sz, sz, sz, vp, vp]

    def dynamic(self, data, graph, entry_point, ids, metric, alpha, window, max_candidates, prune_to,
                threads: int = 0) -> RefDynamic:
        """``MutableVamanaIndex(graph, data, entry_point, distance, ids)`` with every mutation parameter set."""
        d, g, e = _c(data), _c(graph.astype(np.uint32, copy=False)), _c(np.asarray(ids, dtype=np.uint64))
        h = self.lib.svsref_dynamic_create(_code(d), _ptr(d), d.shape[0], d.shape[1], _ptr(g), g.shape[1] - 1,
                                           int(entry_point), METRIC_CODES[metric], _ptr(e), float(alpha), window,
                                           max_candidates, prune_to, threads or effective_cpus())
        if not h:
            raise RuntimeError(self.lib.svsref_dynamic_last_error().decode())
        return RefDynamic(self.lib, h, d.dtype, g.shape[1] - 1)

    def dynamic_build(self, data, ids, metric, alpha, max_degree, window, max_candidates, prune_to,
                      threads: int = 0) -> RefDynamic:
        """``MutableVamanaIndex(parameters, data, ids, distance)`` (the reference's builder, two passes)."""
        d, e = _c(data), _c(np.asarray(ids, dtype=np.uint64))
        h = self.lib.svsref_dynamic_build(_code(d), _ptr(d), d.shape[0], d.shape[1], METRIC_CODES[metric], float(alpha),
                                          max_degree, window, max_candidates, prune_to, _ptr(e),
                                          threads or effective_cpus())
        if not h:
            raise RuntimeError(self.lib.svsref_dynamic_last_error().decode())
        return RefDynamic(self.lib, h, d.dtype, max_degree)
