"""ctypes binding of ``oracle/_ref/libsvsref_dynamic_sq.so``: the reference's ``MutableVamanaIndex`` over
``SQDataset<int8_t / uint8_t>`` (index/vamana/dynamic_index.h, quantization/scalar/scalar.h) compiled from the
unmodified headers (``make -C oracle -f dynamic_sq.mk dynamic_sq``).
TEST INFRASTRUCTURE ONLY: the product package never imports it."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .bindings import HERE, METRIC_CODES, _c, _code, _ptr, effective_cpus


class RefDynamicSQ:
    """The reference's ``MutableVamanaIndex`` over SQ codes behind ``svsref_dynamic_sq_*``; the interface of
    :class:`oracle.dynamic.RefDynamic`, except that ``add`` takes float32 rows and ``export`` also returns the codes."""

    def __init__(self, lib, handle, code_dtype, dim, max_degree):
        self._lib, self._h, self.max_degree = lib, handle, max_degree
        self._code_dtype, self._dim = np.dtype(code_dtype), dim

    def close(self):
        if self._h:
            self._lib.svsref_dynamic_sq_destroy(self._h)
            self._h = None

    __del__ = close

    def _check(self, rc):
        if rc:
            raise RuntimeError(self._lib.svsref_dynamic_sq_last_error().decode())

    def set_params(self, alpha, window, max_candidates, prune_to):
        self._check(self._lib.svsref_dynamic_sq_set_params(self._h, float(alpha), window, max_candidates, prune_to))

    def add(self, points, ids, reuse_empty=False) -> np.ndarray:
        """float32 rows, each encoded by ``SQDataset::set_datum``; returns the slots used."""
        pts = _c(np.asarray(points, dtype=np.float32))
        ids = _c(np.asarray(ids, dtype=np.uint64))
        slots = np.empty(len(ids), dtype=np.uint64)
        self._check(self._lib.svsref_dynamic_sq_add(self._h, _ptr(pts), len(ids), _ptr(ids), int(reuse_empty),
                                                    _ptr(slots)))
        return slots

    def delete(self, ids):
        ids = _c(np.atleast_1d(np.asarray(ids, dtype=np.uint64)))
        self._check(self._lib.svsref_dynamic_sq_delete(self._h, _ptr(ids), len(ids)))

    def consolidate(self):
        self._check(self._lib.svsref_dynamic_sq_consolidate(self._h))

    def compact(self):
        self._check(self._lib.svsref_dynamic_sq_compact(self._h))

    def export(self):
        """(graph uint32[slots][R+1] degree first, status uint8 (0 Empty, 1 Valid, 2 Deleted), external ids
        (2^64 - 1 where not Valid), entry point, codes [slots][dim]) over every slot."""
        n = self._lib.svsref_dynamic_sq_slots(self._h)
        graph = np.zeros((n, self.max_degree + 1), dtype=np.uint32)
        status = np.zeros(n, dtype=np.uint8)
        ext = np.zeros(n, dtype=np.uint64)
        codes = np.zeros((n, self._dim), dtype=self._code_dtype)
        ep = C.c_uint32()
        self._check(self._lib.svsref_dynamic_sq_export(self._h, _ptr(graph), _ptr(status), _ptr(ext), C.byref(ep),
                                                       _ptr(codes)))
        return graph, status, ext, int(ep.value), codes

    def search(self, queries, k, window, capacity=None):
        q = _c(np.asarray(queries, dtype=np.float32))
        capacity = window if capacity is None else capacity
        ids = np.empty((q.shape[0], k), dtype=np.uint64)
        dists = np.empty((q.shape[0], k), dtype=np.float32)
        self._check(self._lib.svsref_dynamic_sq_search(self._h, _ptr(q), q.shape[0], k, window, capacity, _ptr(ids),
                                                       _ptr(dists)))
        return ids, dists


class RefDynamicSQLib:
    """The compiled façade (``oracle/_ref/libsvsref_dynamic_sq.so``)."""
    path = os.path.join(HERE, "_ref", "libsvsref_dynamic_sq.so")

    @classmethod
    def available(cls) -> bool:
        return os.path.exists(cls.path)

    def __init__(self, path=None):
        path = path or self.path
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        self.lib = L = C.CDLL(path)
        sz, vp, f = C.c_size_t, C.c_void_p, C.c_float
        L.svsref_dynamic_sq_last_error.restype = C.c_char_p
        L.svsref_dynamic_sq_create.restype = vp
        L.svsref_dynamic_sq_create.argtypes = [C.c_int, vp, sz, sz, f, f, vp, sz, C.c_uint32, C.c_int, vp, f, sz, sz, sz,
                                               sz]
        L.svsref_dynamic_sq_build.restype = vp
        L.svsref_dynamic_sq_build.argtypes = [C.c_int, vp, sz, sz, f, f, C.c_int, f, sz, sz, sz, sz, vp, sz]
        L.svsref_dynamic_sq_destroy.argtypes = [vp]
        L.svsref_dynamic_sq_set_params.argtypes = [vp, f, sz, sz, sz]
        L.svsref_dynamic_sq_add.argtypes = [vp, vp, sz, vp, C.c_int, vp]
        L.svsref_dynamic_sq_delete.argtypes = [vp, vp, sz]
        L.svsref_dynamic_sq_consolidate.argtypes = [vp]
        L.svsref_dynamic_sq_compact.argtypes = [vp]
        L.svsref_dynamic_sq_slots.restype, L.svsref_dynamic_sq_slots.argtypes = sz, [vp]
        L.svsref_dynamic_sq_export.argtypes = [vp, vp, vp, vp, C.POINTER(C.c_uint32), vp]
        L.svsref_dynamic_sq_search.argtypes = [vp, vp, sz, sz, sz, sz, vp, vp]

    def _codes(self, codes):
        d = _c(codes)
        if d.dtype not in (np.int8, np.uint8):
            raise TypeError("int8 / uint8 codes only")
        return d

    def dynamic(self, codes, scale, bias, graph, entry_point, ids, metric, alpha, window, max_candidates, prune_to,
                threads: int = 0) -> RefDynamicSQ:
        """``MutableVamanaIndex(graph, SQDataset(codes, scale, bias), entry_point, distance, ids)`` with every
        mutation parameter set."""
        d, g, e = self._codes(codes), _c(graph.astype(np.uint32, copy=False)), _c(np.asarray(ids, dtype=np.uint64))
        h = self.lib.svsref_dynamic_sq_create(_code(d), _ptr(d), d.shape[0], d.shape[1], float(scale), float(bias),
                                              _ptr(g), g.shape[1] - 1, int(entry_point), METRIC_CODES[metric], _ptr(e),
                                              float(alpha), window, max_candidates, prune_to,
                                              threads or effective_cpus())
        if not h:
            raise RuntimeError(self.lib.svsref_dynamic_sq_last_error().decode())
        return RefDynamicSQ(self.lib, h, d.dtype, d.shape[1], g.shape[1] - 1)

    def dynamic_build(self, codes, scale, bias, ids, metric, alpha, max_degree, window, max_candidates, prune_to,
                      threads: int = 0) -> RefDynamicSQ:
        """``MutableVamanaIndex(parameters, SQDataset(codes, scale, bias), ids, distance)`` (the reference's builder,
        two passes)."""
        d, e = self._codes(codes), _c(np.asarray(ids, dtype=np.uint64))
        h = self.lib.svsref_dynamic_sq_build(_code(d), _ptr(d), d.shape[0], d.shape[1], float(scale), float(bias),
                                             METRIC_CODES[metric], float(alpha), max_degree, window, max_candidates,
                                             prune_to, _ptr(e), threads or effective_cpus())
        if not h:
            raise RuntimeError(self.lib.svsref_dynamic_sq_last_error().decode())
        return RefDynamicSQ(self.lib, h, d.dtype, d.shape[1], max_degree)
