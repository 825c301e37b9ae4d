"""ctypes wrapper of ``_ref/libsvsref_ivf.so`` (ref/ivf_capi.cpp): the reference's own IVF index behind a test-only
façade.  TEST INFRASTRUCTURE ONLY (see README.md)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref", "libsvsref_ivf.so")


class RefIVF:
    """``assemble_from_clustering`` + ``IVFIndex::search`` of the reference, float32 rows and queries."""

    def __init__(self, path: str = PATH):
        self.lib = C.CDLL(path)
        self.lib.svsref_ivf_last_error.restype = C.c_char_p
        sz, vp = C.c_size_t, C.c_void_p
        self.lib.svsref_ivf_search.argtypes = [vp, sz, sz, C.c_int, vp, sz, vp, vp, sz, sz, sz, vp, vp]

    @staticmethod
    def available() -> bool:
        return os.path.exists(PATH)

    def search(self, data, metric: int, centroids, assignments, queries, k: int, n_probes: int):
        x = np.ascontiguousarray(data, dtype=np.float32)
        c = np.ascontiguousarray(centroids, dtype=np.float32)
        a = np.ascontiguousarray(assignments, dtype=np.uint32)
        q = np.ascontiguousarray(queries, dtype=np.float32)
        ids = np.empty((q.shape[0], k), dtype=np.uint64)
        dists = np.empty((q.shape[0], k), dtype=np.float32)
        rc = self.lib.svsref_ivf_search(x.ctypes.data, x.shape[0], x.shape[1], int(metric), c.ctypes.data, c.shape[0],
                                        a.ctypes.data, q.ctypes.data, q.shape[0], k, n_probes, ids.ctypes.data,
                                        dists.ctypes.data)
        if rc:
            raise RuntimeError(self.lib.svsref_ivf_last_error().decode())
        return ids, dists
