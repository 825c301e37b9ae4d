"""ctypes wrapper of ``_ref/libsvsref_dynamic_ivf.so`` (ref/dynamic_ivf_capi.cpp): the reference's own DynamicIVFIndex
behind a test-only façade.  TEST INFRASTRUCTURE ONLY (see README.md)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libsvsref_dynamic_ivf.so")


class RefDynamicIVF:
    """``assemble_dynamic_from_clustering`` and the mutations and search of the reference's DynamicIVFIndex, float32
    rows and queries."""

    def __init__(self, data, ids, metric: int, centroids, assignments, path: str = PATH):
        self.lib = C.CDLL(path)
        self.lib.svsref_dynivf_last_error.restype = C.c_char_p
        sz, vp = C.c_size_t, C.c_void_p
        self.lib.svsref_dynivf_create.argtypes = [vp, sz, sz, C.c_int, vp, sz, vp, vp, C.POINTER(vp)]
        self.lib.svsref_dynivf_destroy.argtypes = [vp]
        self.lib.svsref_dynivf_destroy.restype = None
        self.lib.svsref_dynivf_add.argtypes = [vp, vp, sz, vp, C.c_int, vp]
        self.lib.svsref_dynivf_delete.argtypes = [vp, vp, sz]
        self.lib.svsref_dynivf_compact.argtypes = [vp]
        self.lib.svsref_dynivf_all_ids.argtypes = [vp, vp, C.POINTER(sz)]
        self.lib.svsref_dynivf_search.argtypes = [vp, vp, sz, sz, sz, vp, vp]
        x = np.ascontiguousarray(data, dtype=np.float32)
        c = np.ascontiguousarray(centroids, dtype=np.float32)
        a = np.ascontiguousarray(assignments, dtype=np.uint32)
        i = np.ascontiguousarray(ids, dtype=np.uint64)
        self.dim = x.shape[1]
        h = C.c_void_p()
        self._check(self.lib.svsref_dynivf_create(x.ctypes.data, x.shape[0], x.shape[1], int(metric), c.ctypes.data,
                                                  c.shape[0], a.ctypes.data, i.ctypes.data, C.byref(h)))
        self.h = h

    @staticmethod
    def available() -> bool:
        return os.path.exists(PATH)

    def _check(self, rc):
        if rc:
            raise RuntimeError(self.lib.svsref_dynivf_last_error().decode())

    def __del__(self):
        if getattr(self, "h", None):
            self.lib.svsref_dynivf_destroy(self.h)
            self.h = None

    def add(self, points, ids, reuse_empty=False) -> list[int]:
        x = np.ascontiguousarray(points, dtype=np.float32)
        i = np.ascontiguousarray(ids, dtype=np.uint64)
        slots = np.empty(len(i), dtype=np.uint64)
        self._check(self.lib.svsref_dynivf_add(self.h, x.ctypes.data, x.shape[0], i.ctypes.data, int(reuse_empty),
                                               slots.ctypes.data))
        return [int(s) for s in slots]

    def delete(self, ids) -> None:
        i = np.ascontiguousarray(ids, dtype=np.uint64)
        self._check(self.lib.svsref_dynivf_delete(self.h, i.ctypes.data, len(i)))

    def compact(self) -> None:
        self._check(self.lib.svsref_dynivf_compact(self.h))

    def all_ids(self) -> np.ndarray:
        n = C.c_size_t(0)
        self._check(self.lib.svsref_dynivf_all_ids(self.h, None, C.byref(n)))
        out = np.empty(n.value, dtype=np.uint64)
        self._check(self.lib.svsref_dynivf_all_ids(self.h, out.ctypes.data, C.byref(n)))
        return out

    def search(self, queries, k: int, n_probes: int):
        q = np.ascontiguousarray(queries, dtype=np.float32)
        ids = np.empty((q.shape[0], k), dtype=np.uint64)
        dists = np.empty((q.shape[0], k), dtype=np.float32)
        self._check(self.lib.svsref_dynivf_search(self.h, q.ctypes.data, q.shape[0], k, n_probes, ids.ctypes.data,
                                                  dists.ctypes.data))
        return ids, dists
